/*
 * frostgpu.h — C-ABI of libfrostgpu.so, the H100 (sm_90a) execution engine for FrostDB's
 * TableScan -> PredicateFilter -> Projection -> HashAggregate/Distinct path.
 *
 * The reference (polarsignals/frostdb, pure Go) has no FFI for this path; its seam is the Go
 * interface physicalplan.ScanPhysicalPlan{Execute,Draw} (query/physicalplan/physicalplan.go:32-35)
 * fed by logicalplan.TableReader.Iterator (query/logicalplan/logicalplan.go:221-241).  Every entry
 * point below names the reference code whose job it takes over.  The cgo binding a FrostDB
 * maintainer would add is shown in INTEGRATION.md and go/physicalplan_gpu.go.
 *
 * Conventions: every function returns int32 status (FGPU_OK == 0, negative == error); the
 * message of the last error on the calling thread is fgpu_last_error().  No exceptions cross the
 * boundary, nothing aborts the process, and the library never calls back into the host from a
 * thread it owns (the only callback, fgpu_match_fn, runs synchronously on the calling thread).
 * All pointers are plain host pointers unless a parameter is explicitly documented as a device
 * pointer.  No torch / C++ types appear in any signature.
 */
#ifndef FROSTGPU_H
#define FROSTGPU_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define FGPU_ABI_VERSION 1

/* ---- status codes -------------------------------------------------------------------------- */
enum {
  FGPU_OK = 0,
  FGPU_ERR_INVALID = -1,     /* bad argument / malformed plan                                     */
  FGPU_ERR_PARQUET = -2,     /* malformed or unsupported Parquet file                             */
  FGPU_ERR_UNSUPPORTED = -3, /* legal FrostDB plan the GPU path does not cover (caller keeps Go)  */
  FGPU_ERR_CUDA = -4,        /* CUDA runtime failure (message has the cudaError string)           */
  FGPU_ERR_NOT_FOUND = -5,   /* unknown table / part / column                                     */
  FGPU_ERR_OOM = -6,         /* device or host allocation failed                                  */
  FGPU_ERR_NO_DEVICE = -7,   /* no CUDA device: the library never falls back to a CPU path        */
  FGPU_ERR_END = -8          /* fgpu_result_next: no more records                                 */
};

/* ---- Arrow C Data Interface (https://arrow.apache.org/docs/format/CDataInterface.html) ------ */
#ifndef ARROW_C_DATA_INTERFACE
#define ARROW_C_DATA_INTERFACE
#define ARROW_FLAG_DICTIONARY_ORDERED 1
#define ARROW_FLAG_NULLABLE 2
#define ARROW_FLAG_MAP_KEYS_SORTED 4
struct ArrowSchema {
  const char* format;
  const char* name;
  const char* metadata;
  int64_t flags;
  int64_t n_children;
  struct ArrowSchema** children;
  struct ArrowSchema* dictionary;
  void (*release)(struct ArrowSchema*);
  void* private_data;
};
struct ArrowArray {
  int64_t length;
  int64_t null_count;
  int64_t offset;
  int64_t n_buffers;
  int64_t n_children;
  const void** buffers;
  struct ArrowArray** children;
  struct ArrowArray* dictionary;
  void (*release)(struct ArrowArray*);
  void* private_data;
};
#endif

/* ---- opaque handles ------------------------------------------------------------------------ */
typedef struct fgpu_ctx fgpu_ctx;       /* one per process per device                            */
typedef struct fgpu_query fgpu_query;   /* a prepared (validated, compiled) plan                 */
typedef struct fgpu_result fgpu_result; /* the records one Execute produced                      */

typedef struct fgpu_config {
  int32_t abi_version; /* FGPU_ABI_VERSION                                                        */
  int32_t device;      /* CUDA device ordinal; one ctx drives exactly one GPU                     */
  int32_t tile_rows;   /* 0 = default; rows decoded per CTA iteration (fixed at build time)        */
  int32_t flags;       /* reserved, 0                                                             */
  uint64_t staging_bytes; /* pinned host staging for uploads; 0 = default (256 MiB)              */
} fgpu_config;

/* ---- plan descriptor: POD mirror of the optimised logicalplan.LogicalPlan ------------------- */

/* logicalplan.Op values, query/logicalplan/expr.go:13-33 (numeric values identical). */
enum {
  FGPU_OP_UNKNOWN = 0, FGPU_OP_EQ, FGPU_OP_NOT_EQ, FGPU_OP_LT, FGPU_OP_LT_EQ, FGPU_OP_GT,
  FGPU_OP_GT_EQ, FGPU_OP_REGEX_MATCH, FGPU_OP_REGEX_NOT_MATCH, FGPU_OP_AND, FGPU_OP_OR,
  FGPU_OP_ADD, FGPU_OP_SUB, FGPU_OP_MUL, FGPU_OP_DIV, FGPU_OP_CONTAINS, FGPU_OP_NOT_CONTAINS
};

/* logicalplan.AggFunc values, query/logicalplan/expr.go:718-729 (numeric values identical).
 * Avg never reaches the engine: Builder.Aggregate rewrites it to Sum+Count+Div
 * (query/logicalplan/builder.go:205-238). */
enum {
  FGPU_AGG_UNKNOWN = 0, FGPU_AGG_SUM, FGPU_AGG_MIN, FGPU_AGG_MAX, FGPU_AGG_COUNT, FGPU_AGG_AVG,
  FGPU_AGG_UNIQUE, FGPU_AGG_AND
};

enum { FGPU_SCALAR_NULL = 0, FGPU_SCALAR_INT64 = 1, FGPU_SCALAR_FLOAT64 = 2, FGPU_SCALAR_STRING = 3 };

typedef struct fgpu_scalar { /* scalar.Scalar of a logicalplan.LiteralExpr                       */
  int32_t type;
  int32_t _pad;
  int64_t i64;
  double f64;
  const uint8_t* bytes; /* FGPU_SCALAR_STRING: not NUL-terminated                                */
  uint64_t len;
} fgpu_scalar;

/* Host-evaluated string matcher for regex leaves (Go's regexp semantics stay in Go): returns
 * non-zero when the dictionary entry matches.  Invoked synchronously, on the thread that called
 * fgpu_query_execute, once per distinct dictionary entry — never per row
 * (replaces the per-row loops of query/physicalplan/regexpfilter.go:85-165). */
typedef int32_t (*fgpu_match_fn)(void* user, const uint8_t* bytes, uint64_t len);

enum { FGPU_EXPR_COLUMN = 1, FGPU_EXPR_DYNCOLUMN = 2, FGPU_EXPR_LITERAL = 3, FGPU_EXPR_BINARY = 4 };

typedef struct fgpu_expr { /* one node of a logicalplan.Expr tree, children by index            */
  int32_t kind;        /* FGPU_EXPR_*                                                            */
  int32_t op;          /* BINARY: FGPU_OP_*                                                      */
  int32_t left, right; /* BINARY: indices into fgpu_plan.exprs                                   */
  const char* name;    /* COLUMN: exact column name; DYNCOLUMN: prefix (matches "name.*",
                          logicalplan.DynamicColumn.MatchColumn expr.go:564)                     */
  fgpu_scalar literal; /* LITERAL                                                                */
  fgpu_match_fn match; /* BINARY with REGEX_MATCH/REGEX_NOT_MATCH: matcher for the pattern       */
  void* match_user;
} fgpu_expr;

typedef struct fgpu_agg { /* logicalplan.AggregationFunction{Func, Expr}                         */
  int32_t func; /* FGPU_AGG_SUM/MIN/MAX/COUNT, FGPU_AGG_UNIQUE over a plain int64 column          */
  int32_t expr; /* index of the aggregated expression (COLUMN or arithmetic BINARY)              */
} fgpu_agg;

enum {
  FGPU_PLAN_AGGREGATE = 1, /* TableScan [-> Filter] [-> Projection] -> Aggregation               */
  FGPU_PLAN_DISTINCT = 2,  /* TableScan [-> Filter] -> Projection -> Distinct                    */
  FGPU_PLAN_FILTER = 3     /* TableScan -> Filter -> Projection(columns): compacted rows          */
};

typedef struct fgpu_plan {
  const char* table;      /* logicalplan.TableScan.TableName                                     */
  int32_t kind;           /* FGPU_PLAN_*                                                         */
  int32_t n_exprs;
  const fgpu_expr* exprs;
  int32_t filter;         /* root of TableScan.Filter (after FilterPushDown), or -1               */
  int32_t n_group_by;     /* AGGREGATE: Aggregation.GroupExprs; DISTINCT/FILTER: output columns   */
  const int32_t* group_by;
  int32_t n_aggs;
  const fgpu_agg* aggs;   /* AGGREGATE: Aggregation.AggExprs                                     */
} fgpu_plan;

typedef struct fgpu_stats {
  uint64_t rows_scanned;      /* rows of visible row groups                                       */
  uint64_t rows_selected;     /* rows that passed the predicate                                   */
  uint64_t groups;            /* result rows                                                     */
  uint64_t algorithmic_bytes; /* stored bytes of the projected column chunks + result bytes      */
  uint64_t metadata_bytes;    /* run directories / tile indexes / LUTs the kernels also read      */
  uint32_t kernel_launches;   /* kernels of this library launched by the Execute                  */
  uint32_t row_groups;
  float scan_kernel_ms;       /* device time of the fused scan kernel (CUDA events)               */
  float total_device_ms;      /* first launch to last result byte on the host                     */
  float h2d_ms;               /* uploads performed inside this Execute (streamed parts)           */
  uint64_t h2d_bytes;
  uint64_t d2h_bytes;
  uint32_t row_groups_pruned; /* ruled out by chunk statistics before upload (index/lsm.go:437)      */
  uint32_t row_groups_runs;   /* scanned by the sorted-run kernel                                   */
  uint32_t row_groups_tiles;  /* scanned by the tile-aggregate kernel (the rest: general scan kernel) */
  uint32_t row_groups_prefix; /* of row_groups_runs: all-pass row groups answered from prefix sums     */
  uint64_t rows_touched;      /* rows of the row groups that survived pruning (what the kernels read)  */
} fgpu_stats;

/* ---- lifecycle ----------------------------------------------------------------------------- */

/* Creates the engine for one GPU: streams, memory pools, pinned staging.  Fails with
 * FGPU_ERR_NO_DEVICE when no CUDA device is usable.  Go side: constructed once by the new
 * physicalplan.Option next to WithOverrideInput (physicalplan.go:279-285). */
int32_t fgpu_init(const fgpu_config* cfg, fgpu_ctx** out);
int32_t fgpu_shutdown(fgpu_ctx* ctx);
const char* fgpu_last_error(void);
int32_t fgpu_abi_version(void);

/* ---- part registry: replaces Table.Iterator / collectRowGroups / LSM.Scan -------------------
 * (table.go:740-868,1179-1242; index/lsm.go:401-454).  A part is one immutable Parquet file as
 * produced by compaction (table.go:1267 compactParts) or one L0 Arrow record (parts/arrow.go). */

enum {
  FGPU_PUT_DEFAULT = 0,
  FGPU_PUT_BORROW_PINNED = 1 /* `file` is page-locked memory that outlives the part: column
                                chunks are not copied at put time but streamed H2D by the
                                queries that project them (the reference reads only projected
                                columns too, optimize.go:36-73)                                  */
};

/* Parses footer + page headers on the host.  FGPU_PUT_DEFAULT then builds every column (run
 * directories, chunk seeds, global dictionary ids) and uploads it, and the caller may free the
 * buffer on return.  FGPU_PUT_BORROW_PINNED keeps the pointer instead: a column is built and
 * uploaded by the first query that projects it, its PLAIN pages DMA'd straight from `file`.
 * DELTA_BINARY_PACKED int64 pages travel encoded and are decoded on the device into the same dense
 * value array as PLAIN pages; a chunk the engine cannot read (compressed, a malformed page, an
 * unsupported encoding) fails only the queries that project its column, with FGPU_ERR_UNSUPPORTED.
 * `tx` is the part's transaction id (parts.Part.TX()). */
int32_t fgpu_part_put_parquet(fgpu_ctx* ctx, const char* table, uint64_t part_id, uint64_t tx,
                              const uint8_t* file, uint64_t len, int32_t flags);

/* L0 Arrow-record part (parts/arrow.go:14-55) through the Arrow C Data Interface; the library
 * calls release() on both structs before returning.  Supported column types: int64, float64,
 * dictionary<uint32|int32, binary|utf8>. */
int32_t fgpu_part_put_arrow(fgpu_ctx* ctx, const char* table, uint64_t part_id, uint64_t tx,
                            struct ArrowSchema* schema, struct ArrowArray* array);

/* Page-locked host memory for parts handed over with FGPU_PUT_BORROW_PINNED (the Go side would
 * write the compacted part straight into such a buffer instead of a bytes.Buffer, table.go:1267). */
int32_t fgpu_host_alloc(uint64_t bytes, void** out);
int32_t fgpu_host_free(void* p);

int32_t fgpu_part_drop(fgpu_ctx* ctx, const char* table, uint64_t part_id);
int32_t fgpu_table_drop(fgpu_ctx* ctx, const char* table);

/* ---- query: replaces physicalplan.Build's TableScan->PredicateFilter->Projection->
 * HashAggregate/Distinction chain (physicalplan.go:287-516; filter.go; aggregate.go; distinct.go)
 * and Synchronizer + final HashAggregate (synchronize.go:16-53, physicalplan.go:438-471). ------ */

int32_t fgpu_query_prepare(fgpu_ctx* ctx, const fgpu_plan* plan, fgpu_query** out);

/* Blocking.  Scans every part of the table with tx <= tx_watermark (lsm.go:416) and produces the
 * final records.  Safe to call from several threads on one ctx: the calls are serialised by the context's mutex and run
 * one after the other on its one stream (contexts on different GPUs, or several contexts on one GPU, run concurrently). */
int32_t fgpu_query_execute(fgpu_ctx* ctx, fgpu_query* q, uint64_t tx_watermark, fgpu_result** out);

/* Next result record as an Arrow struct array (one child per output column).  Ownership passes
 * to the caller through the release callbacks.  Group-by columns are dictionary<uint32, binary>
 * (or int64; a boolean Distinct key such as `value > 0` is a bool column named after its expression, never NULL),
 * aggregate columns are named "sum(value)", "count(value)", ... exactly as
 * aggregate.go:615-618 names them.  Returns FGPU_ERR_END after the last record. */
int32_t fgpu_result_next(fgpu_result* r, struct ArrowSchema* out_schema, struct ArrowArray* out_array);
int32_t fgpu_result_stats(const fgpu_result* r, fgpu_stats* out);
int32_t fgpu_result_free(fgpu_result* r);
int32_t fgpu_query_free(fgpu_query* q);

/* ---- multi-GPU (one process per GPU): the partial -> Synchronizer -> final split -------------
 * (physicalplan.go:438-471).  A rank scans its own parts into a device-resident partial table;
 * the host moves the flat partial buffers between ranks with one collective
 * (ncclAllGather / torch.distributed.all_gather on the device pointer) and any rank merges. */

/* Strings of the table's global dictionary for `column` in id order (id 0 first), as one
 * length-prefixed blob: repeated {uint32 LE length, bytes}.  Call with buf == NULL to size. */
int32_t fgpu_dict_export(fgpu_ctx* ctx, const char* table, const char* column, uint8_t* buf,
                         uint64_t cap, uint64_t* out_len, uint32_t* out_count);
/* Cross-rank id space: interns the given strings (blob format above), in order, into the table's
 * dictionary of `column`.  Every rank preloads the same union list BEFORE putting its parts, so the
 * ids — and therefore the partial tables — agree across ranks.  Entries already present keep their id. */
int32_t fgpu_dict_preload(fgpu_ctx* ctx, const char* table, const char* column,
                          const uint8_t* blob, uint64_t len, uint32_t count);
/* Host-only: the distinct strings of `column` in one Parquet file, in the blob format above, in the
 * order a put of the file interns them: per row group the dictionary page's entries, then the
 * non-dictionary pages' values that are not among them, in order of first occurrence (first-seen order over the
 * file).  Lets a rank contribute its strings to the union without uploading. */
int32_t fgpu_parquet_dict_values(const uint8_t* file, uint64_t len, const char* column,
                                 uint8_t* buf, uint64_t cap, uint64_t* out_len, uint32_t* out_count);

/* Scan only.  `*dev_ptr` is a DEVICE pointer to a position-independent partial table of
 * `*nbytes` bytes.  A dense table (dictionary keys with a small product of cardinalities) has the
 * same size on every rank for the same query + unified dictionaries; a hash table is sized from
 * the rank's own visible rows, so its size can differ between ranks. */
int32_t fgpu_query_execute_partial(fgpu_ctx* ctx, fgpu_query* q, uint64_t tx_watermark,
                                   fgpu_result** out, void** dev_ptr, uint64_t* nbytes);
/* Merges `n` partial tables laid out back to back at DEVICE pointer `gathered` (each `nbytes`
 * long, e.g. the output of an all-gather) into `r` and finalises it.  Every partial must have the
 * size of `r`'s own (FGPU_ERR_INVALID otherwise); a hash-mode merge table is sized for the groups of
 * all `n`.  The collective Execute has no such restriction: it merges hash tables of any size. */
int32_t fgpu_result_merge_partials(fgpu_ctx* ctx, fgpu_result* r, const void* gathered,
                                   uint64_t nbytes, int32_t n);
/* `*out` = 1 when the partial table of `r` merges by element-wise int64 addition (dense table, every
 * aggregate a Count or an integer Sum): the ranks may then all-reduce (SUM) the tables in place over
 * nbytes / 8 int64 words and call fgpu_result_merge_partials(ctx, r, NULL, 0, 0) instead of gathering
 * them — the dense-table reduction of the partial -> final aggregate step (physicalplan.go:438-471). */
int32_t fgpu_result_partial_is_additive(const fgpu_result* r, int32_t* out);

/* ---- the exchange inside the library: peer-mapped mailboxes over NVLink -------------------------
 * The Synchronizer + final HashAggregate of physicalplan.go:438-471 / synchronize.go:16-53 as ONE call per
 * rank: scan -> push the partial table into every rank's mailbox (NVLink stores) -> wait for every rank's
 * flag -> merge -> result, all on the library's stream with a single host synchronisation.  Ranks are
 * contexts: one process per GPU (mailboxes mapped through CUDA IPC) or several contexts in one process
 * (plain peer access); both may be mixed.
 *
 *   1. every rank:  fgpu_comm_export(ctx, rank, n, slot_bytes, handle)      -- allocates this rank's mailbox
 *   2. the caller exchanges the n 128-byte handles (any transport: gloo, a channel, a file)
 *   3. every rank:  fgpu_comm_open(ctx, all_handles)                        -- maps the peers' mailboxes
 *   4. every rank, in the same order: fgpu_query_execute_collective(...)    -- every rank gets the merged result
 *   5. after a barrier of the caller: fgpu_comm_close(ctx)
 * Dictionaries must have been unified with fgpu_dict_preload before the parts were put, exactly as for
 * fgpu_query_execute_partial.  `slot_bytes` bounds the partial table of one query (dense tables:
 * slots * 8 * (1 + stored aggregates)); a larger table fails with FGPU_ERR_UNSUPPORTED. */
#define FGPU_COMM_HANDLE_BYTES 128
int32_t fgpu_comm_export(fgpu_ctx* ctx, int32_t rank, int32_t n_ranks, uint64_t slot_bytes,
                         uint8_t handle[FGPU_COMM_HANDLE_BYTES]);
int32_t fgpu_comm_open(fgpu_ctx* ctx, const uint8_t* all_handles /* n_ranks * FGPU_COMM_HANDLE_BYTES, rank order */);
int32_t fgpu_comm_close(fgpu_ctx* ctx);
/* Collective Execute: every rank of the communicator calls it with the same plan; `*out` holds the merged
 * result on every rank.  A peer that does not arrive within the timeout (FROSTGPU_COMM_TIMEOUT_MS, default
 * 10000) fails the call with FGPU_ERR_CUDA instead of hanging the GPU. */
int32_t fgpu_query_execute_collective(fgpu_ctx* ctx, fgpu_query* q, uint64_t tx_watermark, fgpu_result** out);
/* The same in two halves, for callers that overlap other work with the exchange (and for ranks that share one
 * device, where a rank's flag wait must not be enqueued before its peers have pushed): `begin` scans and pushes
 * this rank's partial table, `end` waits for the peers, merges and finalises `r`. */
int32_t fgpu_query_execute_collective_begin(fgpu_ctx* ctx, fgpu_query* q, uint64_t tx_watermark, fgpu_result** out);
int32_t fgpu_query_execute_collective_end(fgpu_ctx* ctx, fgpu_result* r);

/* ---- standalone K1: decode one column of one part to Arrow buffers on the device and return
 * them on the host (replaces ParquetConverter.Convert, pqarrow/arrow.go:264-373, for tests and
 * for Filter-only consumers). ------------------------------------------------------------------ */
int32_t fgpu_part_decode_column(fgpu_ctx* ctx, const char* table, uint64_t part_id,
                                const char* column, struct ArrowSchema* out_schema,
                                struct ArrowArray* out_array);

/* ---- host-only introspection (works without a GPU; used by the CPU test-suite) --------------- */

/* What the engine decides for a whole row group about the leaf "int64 column <op> literal" from the chunk
 * statistics alone (the decision LSM.Scan's TrueNegativeFilter makes, index/lsm.go:437,
 * expr/binaryscalarexpr.go:84-190): *out_mode = 0 undecided (the kernels evaluate the leaf), 1 every row
 * passes, 2 no row can pass (under a conjunction the row group is skipped). */
int32_t fgpu_rowgroup_leaf_mode(int32_t op, int64_t literal, int32_t has_bounds, int64_t min_value, int64_t max_value,
                                int64_t null_count, int64_t num_values, int32_t* out_mode);

/* Split-block bloom filters (Parquet BloomFilter.md; parquet-go writes one per sorting column,
 * dynparquet/schema.go:1111-1157; checked by expr/binaryscalarexpr.go:104-118): XXH64 of a value's PLAIN encoding, the
 * check and — for tests that build filters — the insert. */
int32_t fgpu_xxhash64(const uint8_t* data, uint64_t len, uint64_t seed, uint64_t* out);
int32_t fgpu_bloom_check(const uint8_t* bitset, uint64_t nbytes, uint64_t hash, int32_t* out_may_contain);
int32_t fgpu_bloom_insert(uint8_t* bitset, uint64_t nbytes, uint64_t hash);

/* One LZ4_RAW block (Parquet codec 7: the LZ4 block format without a frame) that must inflate to exactly `cap` bytes,
 * the size a page header records: validated as the page walk validates a page's block, then inflated into dst (NULL:
 * validate only).  *out_len: the bytes written.  A refused block returns FGPU_ERR_PARQUET naming the rule it breaks. */
int32_t fgpu_lz4_raw_inflate(const uint8_t* src, uint64_t len, uint8_t* dst, uint64_t cap, uint64_t* out_len);

/* The row-group filter's answer for "column == literal" on one row group of a Parquet file, exactly as
 * fgpu_query_execute decides it before anything is uploaded (null count, bloom filter, bounds; LSM.Scan,
 * index/lsm.go:401-454 -> expr/binaryscalarexpr.go:84-128).  lit_type: FGPU_SCALAR_*.  *out: 1 may match, 0 cannot. */
int32_t fgpu_parquet_rowgroup_may_match_eq(const uint8_t* file, uint64_t len, int32_t row_group, const char* column, int32_t lit_type,
                                           int64_t lit_i64, double lit_f64, const uint8_t* lit_bytes, uint64_t lit_len, int32_t* out);

/* Parses a Parquet file exactly as fgpu_part_put_parquet does (footer, page walk, run
 * directories) and writes a JSON description into buf.  Call with buf == NULL to size. */
int32_t fgpu_parquet_describe(const uint8_t* file, uint64_t len, int32_t tile_rows, char* buf,
                              uint64_t cap, uint64_t* out_len);

#ifdef __cplusplus
}
#endif
#endif /* FROSTGPU_H */
