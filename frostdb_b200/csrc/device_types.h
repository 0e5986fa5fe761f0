// Descriptors shared by the host (part store / plan compiler) and the sm_90a kernels.
// Everything here is POD and is copied to the device verbatim.
#pragma once
#include <cstdint>

namespace fgpu {

constexpr int kMaxSlots = 48;    // distinct columns one query may touch
constexpr int kMaxLeaves = 32;   // predicate leaves (one bit each in the per-row leaf mask)
constexpr int kMaxKeys = 40;     // group-by / distinct key columns
constexpr int kMaxAggs = 8;
constexpr int kMaxProg = 48;     // arithmetic ops over all aggregate expressions
constexpr int kMaxFilterProg = 96;
constexpr int kMaxKeyWords = 6;  // packed key = up to 6 x 64 bit
constexpr int kMaxOut = 40;      // projected columns of a rows (filter-only) plan
constexpr int kMaxStagePlain = 4;   // PLAIN columns staged through the shared-memory ring per tile
constexpr int kMaxStageSeeds = 12;  // hybrid streams whose chunk seeds are staged per tile

constexpr uint32_t kNullIdx = 0xffffffffu;

// One run of an RLE/bit-packed hybrid stream (same layout as HostRun).
struct Run {
  uint32_t start;  // first value ordinal of the run within the chunk
  uint32_t off;    // bit-packed: byte offset of the packed payload in the chunk's stream section
  uint32_t val;    // RLE: the repeated value
  uint32_t meta;   // bit0 1 = bit-packed; bits 8..15 bit width
};

enum ChunkKind : uint8_t {
  CK_ABSENT = 0,    // column not in this row group (dynamic column missing): all rows NULL
  CK_PLAIN64 = 1,   // PLAIN int64/double: `values` is a dense 8-byte array of the non-null values
  CK_DICT_STR = 2,  // RLE_DICTIONARY strings: hybrid indices -> lut -> global dictionary id
  CK_DICT64 = 3     // RLE_DICTIONARY int64/double: hybrid indices -> dict64 (8-byte values)
};

// Cursor seed of one hybrid stream for one 128-row chunk: the run that holds the chunk's first value,
// copied out of the run directory so that a warp starts decoding with a single 32-byte read (the
// producer warp stages the 8 seeds of a tile into shared memory with one bulk copy).
struct Seed {
  uint32_t k;      // index of that run in the directory
  uint32_t start;  // = runs[k].start
  uint32_t end;    // = runs[k + 1].start
  uint32_t off;    // = runs[k].off
  uint32_t val;    // = runs[k].val
  uint32_t meta;   // = runs[k].meta
  uint32_t val0;   // value stream: ordinal of the chunk's first value; def stream: non-null values before the chunk
  uint32_t _pad;
};
static_assert(sizeof(Seed) == 32, "seed is one 32-byte sector");

// One column chunk (row group x column) resident in HBM.  All pointers are device pointers into the
// part's single allocation; every section is 128-byte aligned and padded by 16 readable bytes.
struct ChunkDesc {
  uint8_t kind;
  uint8_t has_nulls;  // definition levels stored and at least one NULL
  uint8_t _pad[2];
  uint32_t n_rows;
  uint32_t n_bp_runs; // bit-packed runs in the value directory (0: the chunk is run-length only)
  uint32_t n_values;  // non-null values
  uint32_t n_runs;    // value runs (excluding the sentinel)
  uint32_t n_defruns;
  uint32_t dict_size;
  const uint8_t* values;   // PLAIN64: aligned values; DICT*: concatenated hybrid index streams
  const Run* runs;         // DICT*: run directory (+1 sentinel with start == n_values); CK_DICT_STR: the
                           // value of an RLE run is already the GLOBAL dictionary id
  const Seed* seeds;       // DICT*: one per 128-row chunk
  const uint8_t* def;      // concatenated definition-level hybrid streams (has_nulls)
  const Run* def_runs;     // (+1 sentinel with start == n_rows)
  const Seed* def_seeds;   // has_nulls: one per 128-row chunk (val0 = non-null values before the chunk)
  const uint32_t* lut;     // CK_DICT_STR: chunk dictionary index -> global dictionary id (bit-packed runs)
  const int64_t* dict64;   // CK_DICT64: chunk dictionary values (raw 8 bytes each)
  // CK_DICT_STR whose value AND definition-level streams are run-length only (sorted parts): one directory in
  // ROW space, val = global dictionary id or 0xffffffff for NULL (+1 sentinel with start == n_rows), with
  // its per-128-row seeds.  A column without NULLs aliases runs / seeds.  Null: not available.
  const Run* row_runs;
  const Seed* row_seeds;
  uint32_t n_row_runs;
  uint32_t _pad_rr;
};

enum SlotType : uint8_t { ST_I64 = 0, ST_F64 = 1, ST_DICT = 2 };

enum LeafMode : uint8_t { LM_EVAL = 0, LM_ALL = 1, LM_NONE = 2 };

// Predicate leaf "column op literal" (binaryscalarexpr.go:41-152), canonicalised by the host:
// numeric comparisons become "value inside the inclusive range [lo, hi]", optionally negated
// (== v -> [v,v]; != v -> not [v,v]; < v -> [min, v-1]; >= v -> [v, max]; ...), so the kernels
// run one branch-free range test per leaf, and conjunctions of comparisons on the same column
// (timestamp >= a AND timestamp < b) are intersected into ONE leaf.
struct LeafDesc {
  uint8_t slot;
  uint8_t op;         // original logicalplan.Op (dictionary leaves)
  uint8_t cmp_float;  // compare as double (float column, or int column against float literal)
  uint8_t neg;        // numeric: select rows OUTSIDE the range
  uint32_t _pad2;
  int64_t lo_i, hi_i;
  double lo_f, hi_f;
};

// Per (row group, leaf): how the leaf behaves on that row group.
struct LeafRt {
  uint8_t mode;         // LeafMode; ALL/NONE encode the missing-column rules (binaryscalarexpr.go:47-73)
  uint8_t null_result;  // dictionary leaves: result for NULL rows (== NULL selects nulls, :205-212)
  uint8_t _pad[6];
  const uint8_t* lut;   // dictionary leaves: result per GLOBAL dictionary id
};

struct KeyDesc {
  uint8_t slot;
  uint8_t is_int64;  // key is a raw int64 column (takes a whole 64-bit word)
  uint8_t word;      // packed mode: which 64-bit key word
  uint8_t shift;     // packed mode: bit offset inside the word
  uint32_t bits;     // packed mode: field width
  uint32_t dense_stride;  // dense mode: multiplier of (gid + 1)
  uint8_t prog_off, prog_len;  // computed int64 key ((timestamp / 1000) * 1000): its program in QueryDesc::prog (prog_len > 0);
                               // boolean key: its program in BoolKeys::prog
  uint8_t is_bool;   // boolean key (Distinct(..., value > 0)): code 1 false, 2 true in a 2-entry code key (radix 3)
  uint8_t _pad;
};
static_assert(sizeof(KeyDesc) == 16, "KeyDesc");

enum ProgOpCode : uint8_t { PO_LOAD = 0, PO_CONST = 1, PO_ADD = 2, PO_SUB = 3, PO_MUL = 4, PO_DIV = 5 };
struct ProgOp {
  uint8_t op;
  uint8_t slot;
  uint8_t _pad[6];
  int64_t imm;  // PO_CONST: int64 or the bits of a double
};

// Unique(int64) is two stored cells, a Min then a Max of the same column, in which a NULL row counts as INT64_MIN and as
// INT64_MAX: the group's value is the one both cells hold, NULL when they differ (aggregate.go:677-730).  Every reducer,
// merge and exchange treats them as the Min and Max they are; only the scan's input and the finalize read `unique`.
enum UniqueCell : uint8_t { UC_NONE = 0, UC_LO = 1, UC_HI = 2 };

struct AggDesc {
  uint8_t func;      // logicalplan.AggFunc value (a Unique cell: Min or Max)
  uint8_t is_float;  // expression evaluates in float64
  uint8_t prog_off;
  uint8_t prog_len;
  uint8_t unique;    // UniqueCell; the UC_HI cell directly follows its UC_LO cell
  uint8_t _pad[3];
};

enum TableMode : int32_t { TM_DENSE = 0, TM_HASH = 1 };
enum FilterKind : int32_t { FK_PROGRAM = 0, FK_AND = 1, FK_OR = 2 };  // conjunction / disjunction of leaves: one mask test

// Everything one launch of the fused scan kernel needs.
struct QueryDesc {
  int32_t n_slots, n_leaves, n_keys, n_aggs;
  int32_t n_filter_prog;  // 0 = no filter
  int32_t table_mode;
  int32_t key_words;
  int32_t tile_rows;
  int32_t n_rg;
  uint32_t n_tiles;
  uint32_t table_slots;  // dense: number of slots; hash: capacity (power of two)
  int32_t filter_kind;   // FilterKind
  uint32_t filter_mask;  // FK_AND / FK_OR: the participating leaf bits
  int32_t n_out;         // rows plan: projected columns
  int32_t n_stage_plain, n_stage_seeds, n_stages;  // staged PLAIN slices / seeds per vector (scan kernel)
  int32_t vl;            // rows per warp vector (scan kernel)
  int32_t fast_ok;       // query shape qualifies for the fused register-only pass (vec_fast)
  int32_t n_ring;        // ring depth per warp
  uint32_t slot_bytes;   // bytes of one ring slot
  uint32_t wr_bytes;     // per-warp shared-memory region: size and section offsets
  uint32_t wr_ring, wr_act, wr_leaf, wr_slot, wr_keyw, wr_tmp1, wr_tmp2, wr_acc, wr_cdesc, wr_clrt, wr_fplan, wr_iplan;
  uint8_t stage_plain_slot[kMaxStagePlain];   // staged PLAIN buffer p holds this slot
  uint8_t stage_seed_slot[kMaxStageSeeds];    // staged seed block t belongs to this slot ...
  uint8_t stage_seed_is_def[kMaxStageSeeds];  // ... and is its definition-level stream (1) or value stream (0)
  int8_t slot_plain_stage[kMaxSlots];         // slot -> staged PLAIN buffer, -1 = read from HBM
  int8_t slot_seed_stage[kMaxSlots][2];       // slot -> staged seed block of [0] values, [1] def levels, -1 = read from HBM
  uint8_t slot_type[kMaxSlots];
  uint8_t out_slot[kMaxOut];
  uint8_t slot_used_by_leaf[kMaxSlots];
  uint8_t filter_prog[kMaxFilterProg];  // postfix: 0..31 push leaf; 0x80 AND; 0x81 OR
  LeafDesc leaves[kMaxLeaves];
  KeyDesc keys[kMaxKeys];
  AggDesc aggs[kMaxAggs];
  ProgOp prog[kMaxProg];
  // per row group tables
  const ChunkDesc* chunks;        // [n_rg][n_slots]
  const LeafRt* leaf_rt;          // [n_rg][n_leaves]
  const uint32_t* rg_first_tile;  // [n_rg + 1]
  const uint32_t* rg_rows;        // [n_rg]
  // aggregate table
  unsigned long long* t_rows;  // rows per slot (also every Count aggregate)
  long long* t_agg[kMaxAggs];  // per aggregate, int64 or double bits
  uint32_t* t_tag;             // hash mode: 0 empty, 1 locked, else fingerprint|2
  unsigned long long* t_keys;  // hash mode: [capacity][key_words]
  unsigned long long* counters;  // [0] rows selected, [1] table overflow flag, [2] tile ticket (rows plan)
  // rows plan outputs
  void* out_data[kMaxOut];       // int32 global ids (dictionary columns) or raw 8-byte values
  uint8_t* out_valid[kMaxOut];   // numeric columns: 0/1 per output row
  unsigned long long* tile_state;  // [n_tiles] decoupled look-back state
  const struct BoolKeys* bool_keys;  // boolean Distinct keys (k_scan only); null: the plan has none
};
// Every kernel holds QueryDesc in shared memory or takes it by value as a kernel parameter: keep it inside 4 KB.
static_assert(sizeof(QueryDesc) <= 4096, "QueryDesc grew past 4 KB");

// The boolean keys of a Distinct (`Distinct(labels.a, value > 0)`, project.go:397-467): each key is a postfix program
// over its own predicate leaves, which are compiled like the filter's but never select or drop a row.  The block is
// uploaded with the plan; k_scan copies it, and the key leaves' LeafRt of the row group it works on, into the warp's
// shared-memory region at wr_keys.
struct BoolKeys {
  int32_t n_leaves;  // key leaves (filter leaves + key leaves <= kMaxLeaves)
  uint32_t wr_keys;  // offset of the per-warp copy: [BoolKeys][LeafRt x n_leaves]
  const LeafRt* leaf_rt;  // [n_rg][n_leaves]
  uint8_t prog[kMaxFilterProg];  // postfix programs of every key (KeyDesc::prog_off / prog_len): 0..31 push leaf; 0x80 AND; 0x81 OR
  LeafDesc leaves[kMaxLeaves];
};

// Dense/hash table -> compacted result rows.
// One PLAIN page payload to move from the raw chunk bytes (copied from the host in ONE transfer per column
// chunk, page headers and level bytes included) to its place in the dense value array (k_gather_pages).
struct PageCopy {
  uint64_t src_off;  // byte offset inside the staging buffer (any alignment)
  uint64_t dst_off;  // byte offset inside the column image (8-byte aligned)
  uint64_t len;      // multiple of 8
};

// One cursor-seed array to derive on the device from an uploaded run directory (k_make_seeds): the
// seeds are 32 bytes per 128 rows, far more than the directory of a sorted column, so they are computed
// where they are used instead of being built and copied by the host.  Offsets are relative to the
// column image.
struct SeedJob {
  uint64_t runs_off;   // Run[n_runs + 1] (sentinel included)
  uint64_t seeds_off;  // Seed[n_chunks] to fill
  uint64_t val0_off;   // uint32[n_chunks]: values before each 128-row chunk (nullable columns); ~0: chunk * 128
  uint32_t n_runs, total, n_chunks, is_def;
};

// ---- non-dictionary string pages interned at upload (intern_strings.cu) ------------------------------------
// One column chunk of an intern batch: its PLAIN / DELTA_LENGTH_BYTE_ARRAY / DELTA_BYTE_ARRAY string values
// (validated by the host's page walk) and its open-addressing table, power-of-two capacity of at least twice its values.
// A value is addressed in one of two ways: `len` null (PLAIN pages only): `off` is the offset of its 4-byte length
// prefix; else `off` is its start and `len` its length.  DELTA_BYTE_ARRAY values start at `rb0` or above: k_str_unfront
// rebuilds them there, behind the file bytes.
struct StrChunk {
  uint8_t* bytes;            // the chunk's value regions (a copy of the file bytes), then its rebuilt values
  const uint32_t* off;       // per value: offset of its length prefix, or its start, in `bytes`
  const uint32_t* len;       // per value: its length; null: a length prefix precedes it
  unsigned long long* keys;  // per slot: (hash >> 32) << 32 | representative value index; ~0: empty
  uint32_t* first;           // per slot: smallest value index; after k_str_compact: the slot's rank among the used slots
  uint32_t* slot;            // per value: its slot
  uint32_t* out_first;       // k_str_compact: first value index per rank (page-locked host memory)
  const uint32_t* pre;       // DELTA_BYTE_ARRAY values: prefix length, in page order (null: the chunk has none)
  const uint32_t* suf;       //   start of the suffix in `bytes`
  const uint32_t* wmin;      //   least prefix length of each window of 32 values of a page
  uint8_t* out_rebuilt;      // k_str_gather: the rebuilt region, as `bytes` + rb0 holds it, where distinct values go
                             //   (page-locked host memory; null: the chunk has no DELTA_BYTE_ARRAY values)
  uint32_t n, mask;          // values; capacity - 1
  uint32_t v0, s0;           // values / slots of the batch's chunks before this one
  uint32_t rb0, _pad;        // start of the rebuilt values in `bytes` (~0: none)
};

// A run of at most kFrontSeg values of one DELTA_BYTE_ARRAY page, which one warp of k_str_unfront rebuilds.
struct StrFrontJob {
  uint32_t chunk;       // in the batch
  uint32_t v0, d0, w0;  // the page's first value, its index in pre / suf, its first window in wmin
  uint32_t seg, n;      // the run's first value, relative to the page; its values
};

// One PLAIN string page whose chunk-local indices k_str_codes packs, LSB first, into the hole its page owns.
struct StrCodeJob {
  uint8_t* dst;           // the hole: ceil(n / 8) * w bytes (an image offset until the image is resident)
  const uint32_t* slot;   // per value of the page: its slot
  const uint32_t* rank;   // per slot of its chunk: rank
  const uint32_t* code;   // per rank of its chunk: chunk-local index
  uint32_t n, w;          // values; bits per index (1 .. 24)
  uint32_t g0, _pad;      // 8-value groups of the launch's jobs before this one
};

// ---- DELTA_BINARY_PACKED int64 pages decoded at upload (delta_int64.cu) --------------------------------------
// One page of a column upload: its values are the page's first value, then one value per delta, written to `dst`.
// The upload's pages are listed in order of g0, the ordinal of the page's first 32-value group among the upload's groups.
struct DbpPage {
  unsigned long long* dst;  // its n dense values (in the column image)
  unsigned long long src;   // offset of its stream in the staging buffer
  unsigned long long first; // its first value
  uint32_t n, g0;           // values (>= 1); first group
  uint32_t mb0, per_mb;     // its first miniblock in the upload's list; values per miniblock (clamped to 2^32 - 1)
};

// One miniblock of a page holding values: the deltas of the page's values 1 + k for k in [m * per_mb, (m + 1) * per_mb),
// m its index within the page.
struct DbpMini {
  unsigned long long min_delta;
  uint32_t off;    // byte offset of its packed deltas from the page's stream start
  uint32_t width;  // 0 .. 64
};
constexpr int kDbpGroupsPerCta = 32;  // one warp per 32-value group: a CTA covers 1 024 values

// ---- LZ4_RAW value pages inflated at upload (lz4_pages.cu) ---------------------------------------------------
// One PLAIN INT64 / DOUBLE page whose LZ4_RAW block the host validated: the block sits in the upload's staging buffer,
// its first `out_len` inflated bytes are the page's dense values (a hole in the column image).
struct Lz4Job {
  unsigned char* dst;      // its hole in the column image
  unsigned long long src;  // offset of its block in the staging buffer
  uint32_t len;            // bytes of the block
  uint32_t out_len;        // bytes of the hole (8 per non-null value)
};
constexpr int kLz4WarpsPerCta = 4;  // one warp per page

// ---- sorted-run scan (k_runs_tma): the plan shape of compacted parts -----------------------------------
// Row groups whose filter columns and aggregate inputs are PLAIN non-null int64 and whose group-key
// columns are run-length only (sorted parts) are scanned by a dedicated kernel that walks the key run
// directories with warp-uniform cursors.  The host lists those row groups here; the rest of the table
// goes through the general scan kernel into the same aggregate table.
constexpr int kRunsLeaves = 2, kRunsKeys = 3, kRunsAggs = 3, kRunsCols = kRunsLeaves + kRunsAggs;
constexpr int kRunsPreds = 2;  // dictionary-column leaves evaluated once per run (result byte per dictionary id)
constexpr int kRtConsumerWarps = 8;                         // k_runs_tma: consumer warps per CTA (most; 4 / 8)
constexpr int kRtMaxThreads = (kRtConsumerWarps + 1) * 32;  // + one producer warp
constexpr int kRtDirMax = 128;                              // most directory entries staged per cursor column and tile

// Staged column c of a row group: uint{8,16,32,64}(value - base) per row, 1 << lg bytes each (a frame-of-reference
// image, or the 8-byte PLAIN values with base 0), at byte soff of the stage's column region.  A decided leaf's column
// in a row group that is not all_pass is not staged (RunsRg::col[c] null): it takes a staged column's entry (stand-in).
struct alignas(16) RunsCol {
  uint32_t soff, lg;
  long long base;
};

struct RunsRg {
  uint32_t n_rows;
  uint32_t all_pass;  // 1: the chunk statistics decided every leaf (all rows pass); the leaf columns are not staged
  long long lo[kRunsLeaves], hi[kRunsLeaves];  // inclusive bounds of the (fused) range leaves for this row group
  const uint8_t* col[kRunsCols];               // the staged columns (distinct leaf and aggregate inputs): image or values
  const Run* runs[kRunsKeys];                  // run directory of every group-key column (dictionary ids premapped)
  const Seed* seeds[kRunsKeys];                // cursor seeds, one per kIndexRows rows
  // dictionary leaves (== / != / contains / regex on a run-length column): row-space directory + seeds of the
  // leaf's column and the leaf's result per GLOBAL dictionary id; runs == null: decided for this row group (passes)
  const Run* pred_runs[kRunsPreds];
  const Seed* pred_seeds[kRunsPreds];
  const uint8_t* pred_lut[kRunsPreds];
  uint32_t n_runs[kRunsKeys];                  // entries of every key directory (the sentinel not counted)
  uint32_t pred_n_runs[kRunsPreds];
  uint32_t tile_rows;                          // rows per tile in this row group (about 32 KB of staged column data)
  RunsCol cl[kRunsCols];                       // layout of every staged column (copied into each stage header)
};
static_assert(sizeof(RunsRg) % 16 == 0, "RunsRg::cl is copied with TMA");

struct RunsDesc {
  uint32_t n_rg, n_spans;
  uint32_t block_rows;   // rows per prefetch block (multiple of 128)
  uint32_t span_blocks;  // blocks per span: a span is the contiguous piece of a row group one warp takes per turn
  uint32_t n_ring, n_cols;
  uint32_t leaf_col[kRunsLeaves], agg_col[kRunsAggs];  // index into RunsRg::col
  uint32_t stride[kRunsKeys];                           // dense-table stride of every key
  uint32_t agg_func[kRunsAggs];                         // AggFunc | is_float << 8 (general-reducer instances)
  uint32_t n_pred;                                      // dictionary leaves (conjunction with the range leaves)
  uint32_t pred_null[kRunsPreds];                       // their result for NULL rows (== NULL selects NULLs)
  // k_runs_tma (runs_tma.cu): block_rows = rows per tile, span_blocks = tiles per span, n_ring = ring stages
  uint32_t dir_entries;                                 // directory entries staged per cursor column and tile
  uint32_t stage_bytes, col_off;                        // bytes of one ring stage; offset of the staged columns inside it
  uint32_t n_consumers, consumers_log2;                 // consumer warps per CTA
  uint32_t _pad_rt;
  const RunsRg* rgs;
  const uint32_t* rg_first_span;  // [n_rg + 1]
  unsigned long long* t_rows;
  long long* t_agg[kRunsAggs];
  unsigned long long* counters;
};

// ---- all-pass sorted row groups from prefix sums (k_runs_prefix, runs_prefix.cu) ----------------------------
// A sorted-run row group whose filter the chunk statistics decided (every row passes) and whose stored aggregates are
// all Sum(int64) is answered from the run directories of its key columns and the exclusive prefix sums of its Sum inputs
// (ensure_narrow): the rows [b, e) of one group add P[e] - P[b] and e - b.
//
// The segments [b, e) (maximal stretches of one row group with one dense slot) depend only on the key directories and
// the dense strides, so a build step (k_prefix_segs) enumerates them once per compiled plan, from windows the host cuts,
// into a table grouped by slot; every Execute then folds each slot's list (k_runs_prefix).
struct PrefixRg {
  uint32_t n_rows;
  uint32_t _pad;
  const long long* pre[kRunsAggs];  // P[0 .. n_rows] of every Sum input, P[i] = v[0] + ... + v[i-1] modulo 2^64
  const Run* runs[kRunsKeys];       // row-space run directory of every key column (+ sentinel)
  const Seed* seeds[kRunsKeys];     // its cursor seeds, one per kIndexRows rows
  uint32_t n_runs[kRunsKeys];
  uint32_t _pad2;
};

struct alignas(16) PrefixWin {
  uint32_t rg, r0, rows, _pad;  // rows [r0, r0 + rows) of row group rg
};

struct PrefixSeg {
  uint32_t rg, b, e;  // rows [b, e) of row group rg (index into the launch's PrefixRg array)
};

// Build step: count the segments of every slot (cnt, zeroed), exclusive scan into seg_off, then scatter them (cnt
// counts down to 0 again).
struct PrefixBuildDesc {
  uint32_t n_win, nk;
  uint32_t stride[kRunsKeys];  // dense-table stride of every key
  const PrefixRg* rgs;
  const PrefixWin* wins;
  uint32_t* cnt;           // [table_slots + 1]
  const uint32_t* seg_off;  // [table_slots + 1]
  PrefixSeg* seg;
};

// Execute: every slot of the dense table gets its rows and Sums stored (0 without segments), and counters[0..9] are
// set (rows selected = all rows of the prefix row groups), so this launch replaces k_table_init.
struct PrefixDesc {
  uint32_t n_slots, na;
  uint32_t group_log2;  // lanes per slot: 1 << group_log2 up to 32; above 5: a CTA per slot
  uint32_t _pad;
  unsigned long long all_rows;
  const PrefixRg* rgs;
  const uint32_t* seg_off;
  const PrefixSeg* seg;
  unsigned long long* t_rows;
  long long* t_agg[kRunsAggs];
  unsigned long long* counters;
};

// ---- filter-only plans over PLAIN columns (k_take_*, take_rows.cu) -----------------------------------
constexpr int kTakeLeaves = 2, kTakeOut = 4;
constexpr int kTakePreds = 2;  // dictionary-column leaves (==, !=, contains, regex, == NULL) evaluated from flat codes

struct TakeRg {
  uint32_t n_rows;
  uint32_t all_pass;  // 1: statistics decided every leaf (all rows pass): the span is a plain copy
  long long lo[kTakeLeaves], hi[kTakeLeaves];
  const uint8_t* leaf_col[kTakeLeaves];  // PLAIN int64 values of every leaf's column (null: decided for this row group)
  const uint8_t* out_col[kTakeOut];      // PLAIN 8-byte values of every projected column
  // dictionary leaves: flat code array of the leaf's column (k_flatten; null: decided, passes) and the leaf's result
  // byte per GLOBAL dictionary id
  const uint8_t* pred_codes[kTakePreds];
  const uint8_t* pred_lut[kTakePreds];
  uint8_t pred_w[kTakePreds], pred_bias[kTakePreds], pred_null[kTakePreds];  // bits per code; 1: code = id, 0: code = id + 1 (0 = NULL); result for NULL rows
  uint8_t _pad_p[8 - (3 * kTakePreds) % 8];
};

struct TakeDesc {
  uint32_t n_rg, n_spans, span_blocks, nl, n_out, np;
  const TakeRg* rgs;
  const uint32_t* rg_first_span;      // [n_rg + 1]
  unsigned long long* span_count;     // [n_spans + 1]: passing rows per span, then their exclusive prefix
  unsigned long long* total;          // rows that passed (the query's counters[0])
  long long* out_data[kTakeOut];
};

// ---- tile aggregate (k_tile_agg, tile_agg.cu): unsorted / short-run / nullable keys -------------------------
// Row groups the sorted-run kernel cannot take (bit-packed or short-run key columns, NULLs in the keys, fresh
// L0 records) are scanned CTA-cooperatively: one producer warp stages TILES of every projected column into a
// shared-memory ring with TMA bulk copies (cp.async.bulk + mbarrier), the consumer warps aggregate the tile
// into a CTA-private shared-memory table with 32-bit shared atomics and the table is folded into the global
// one once per CTA.  Dictionary columns are read as FLAT CODE arrays: fixed-width codes (global dictionary
// id, or id + 1 with 0 = NULL) derived once per column chunk on the device from the stored hybrid streams
// (k_flatten), so that a tile of any column is one contiguous, 128-byte aligned byte range.
constexpr int kTaPlain = 4;   // staged PLAIN columns (distinct leaf + aggregate inputs)
constexpr int kTaCodes = 6;   // staged flat-code columns (keys + dictionary-leaf columns)
constexpr int kTaLeaves = 3;  // range leaves (conjunction)
constexpr int kTaPreds = 3;   // dictionary leaves (conjunction)
constexpr int kTaKeys = 4;
constexpr int kTaAggs = 4;
constexpr int kTaConsumerWarps = 24;
constexpr int kTaThreads = (kTaConsumerWarps + 1) * 32;  // + one producer warp

struct TileAggRg {
  uint32_t n_rows;
  uint32_t _pad;
  long long lo[kTaLeaves], hi[kTaLeaves];  // inclusive bounds (bits of a double when the leaf compares as float)
  const uint8_t* plain[kTaPlain];          // PLAIN value arrays (null: the column is not read in this row group)
  const uint8_t* codes[kTaCodes];          // flat code arrays (null: column absent, every row NULL)
  const uint8_t* pred_lut[kTaPreds];       // result byte per GLOBAL dictionary id (null: the leaf is decided, passes)
  uint8_t code_w[kTaCodes];                // bits per code
  uint8_t code_bias[kTaCodes];             // 1: chunk without NULLs, code = id; 0: code = id + 1, 0 = NULL
  uint8_t leaf_skip[kTaLeaves];            // 1: decided by statistics / missing-column rules (passes)
  uint8_t _pad2[8 - (2 * kTaCodes + kTaLeaves) % 8];
};
static_assert(sizeof(TileAggRg) % 8 == 0, "copied word-wise into the stage header");

struct TileAggDesc {
  uint32_t n_rg, n_tiles, tile_rows, n_stages, slot_bytes;
  uint32_t n_plain, n_codes;
  uint32_t plain_off[kTaPlain], code_off[kTaCodes];  // byte offsets inside a ring slot
  uint32_t nl, leaf_plain[kTaLeaves], leaf_flags[kTaLeaves];  // flags: 1 compare as double, 2 column is double, 4 negate
  uint32_t np, pred_code[kTaPreds], pred_null[kTaPreds];
  uint32_t nk, key_code[kTaKeys], key_stride[kTaKeys];
  uint32_t na, agg_plain[kTaAggs], agg_func[kTaAggs];  // AggFunc | is_float << 8
  uint32_t table_slots;
  uint32_t rep_log2;             // shared-memory table: every slot has 1 << rep_log2 replicas (lane & (R - 1))
  uint32_t smem_table;           // 0: atomics go to the global table directly
  uint32_t cell_off[kTaAggs];    // shared-memory table: byte offset of the aggregate's cell array (behind the counts)
  uint32_t cell64[kTaAggs];      // 1: 64-bit cells (Min / Max / float64), 0: low word of an int64 Sum
  uint32_t table_bytes;          // shared-memory table bytes
  uint32_t chunk_tiles;          // consecutive tiles a CTA takes per turn
  uint32_t keys8;                // every key code column of this launch is 8 bits wide
  uint32_t sums_fit32;           // chunk statistics prove that no int64 Sum leaves 32 bits inside one CTA
  const TileAggRg* rgs;
  const uint32_t* rg_first_tile;  // [n_rg + 1]
  unsigned long long* t_rows;
  long long* t_agg[kTaAggs];
  unsigned long long* counters;
};

// One column chunk to turn into a flat code array (k_flatten).
struct FlatJob {
  ChunkDesc chunk;     // resident hybrid image
  uint8_t* out;        // flat codes, 128-byte aligned, padded
  uint32_t w, bias;
  uint32_t first_block;  // prefix over the jobs of one launch: 128-row blocks before this job
  uint32_t _pad;
};

// One PLAIN non-null int64 column chunk to restage as a frame-of-reference image and / or an exclusive prefix-sum image
// (k_chunk_minmax, then k_narrow).
struct NarrowJob {
  const long long* src;  // resident values
  uint8_t* out;          // k_narrow: uint{8,16,32}(v - base) per row, 128-byte aligned, padded (w == 0: none)
  long long* pre;        // k_narrow: P[0 .. n_rows], P[i] = v[0] + ... + v[i-1] modulo 2^64 (null: none)
  long long base;        // k_narrow: the chunk minimum
  uint32_t n_rows, w;    // rows; k_narrow: bytes per row
  uint32_t first_block;  // prefix over the jobs of one launch: kNarrowRows-row blocks before this job
  uint32_t sum_block;    // k_narrow: this job's first block in k_chunk_minmax's numbering (its block sums)
};
constexpr uint32_t kNarrowRows = 4096;

constexpr int kMaxRanks = 16;  // GPUs of one node exchanging partial tables (comm.cu)

// Dense table -> compacted result columns for the cached Execute path (k_finalize_dense): dictionary indices as
// uint32 (0xffffffff = NULL), aggregates as raw 8 bytes, so that the host only copies columns.
struct DenseOut {
  uint32_t table_slots, max_out, n_keys, n_aggs;
  uint32_t stride[kMaxKeys], radix[kMaxKeys];
  const unsigned long long* t_rows;
  const long long* t_agg[kMaxAggs];  // null: Count (the row count)
  const unsigned long long* counters;  // the query's counters: [0..3] travel in the header
  // Collective Execute (n_src > 0): the table to compact is the fold of n_src partial tables sitting in this rank's
  // mailbox; the kernel first waits for every peer's flag (the reference's Synchronizer + final aggregate in one
  // launch).  Layout of a partial table: [rows S x 8][stored aggregates S x 8 each, agg_pos says which].
  int32_t n_src, _pad_src;
  const uint8_t* src[kMaxRanks];
  const unsigned long long* flags;      // this rank's flags of the current set: {seq, bytes} per rank
  unsigned long long seq, bytes, timeout_ns;
  unsigned long long* err;              // the query's counters[3]: 1 timeout, 2 table shapes differ
  uint8_t agg_func[kMaxAggs], agg_is_float[kMaxAggs];
  uint8_t agg_unique[kMaxAggs];         // UniqueCell: a UC_HI cell's column holds the validity bytes of its UC_LO cell's
  int8_t agg_pos[kMaxAggs];             // index among the stored aggregates, -1: Count (= rows)
  uint32_t* hdr;  // 256 bytes of device memory, zero between launches (see k_finalize_dense)
  uint8_t* out;   // device or page-locked host memory: [header 256 B: count u32 @0, counters u64 x4 @32, any_null u32 per key @64][n_keys x max_out u32 (8-byte aligned)][n_aggs x max_out i64]
};

// ---- partial-table exchange between the GPUs of one node (comm.cu) ---------------------------------------
struct CommPush {
  unsigned int* done;                  // CTAs that finished their copies (the last one raises the flags); left zero
  const uint8_t* src;                  // this rank's partial table
  unsigned long long bytes;            // multiple of 16
  unsigned long long seq;
  int32_t n, _pad;
  uint8_t* dst[kMaxRanks];             // slot [my rank] of the current set in every rank's mailbox
  unsigned long long* flag[kMaxRanks]; // flag pair {seq, bytes} [my rank] of the current set in every rank's mailbox
};
struct CommWait {
  const unsigned long long* flags;     // this rank's flags of the current set: {seq, bytes} per rank
  unsigned long long seq, bytes, timeout_ns;  // bytes: what every rank must have pushed (dense tables); 0: no check
  unsigned long long* counters;        // the query's counters: [3] = 1 timeout, 2 table shapes differ
  int32_t n, _pad;
};
struct CommMerge {
  const uint8_t* src[kMaxRanks];       // the slots of the current set in this rank's mailbox
  int32_t n, _pad;
};

struct FinalizeDesc {
  int32_t table_mode, key_words, n_keys, n_aggs;
  uint32_t table_slots;
  uint32_t max_out;
  KeyDesc keys[kMaxKeys];
  uint32_t dense_radix[kMaxKeys];  // dense mode: (card + 1) per key
  const unsigned long long* t_rows;
  const long long* t_agg[kMaxAggs];
  const uint32_t* t_tag;
  const unsigned long long* t_keys;
  // outputs
  long long* out_keys;  // [n_keys][max_out] : gid+1 code (0 = NULL) or raw int64
  long long* out_aggs;  // [n_aggs][max_out]
  unsigned long long* out_rows;  // [max_out]
  unsigned int* out_count;
  uint8_t agg_unique[kMaxAggs];  // as DenseOut::agg_unique
};

}  // namespace fgpu
