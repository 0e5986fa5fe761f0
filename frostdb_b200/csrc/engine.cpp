// libfrostgpu host engine: context, part registry uploads, plan compilation, execution, result
// export, and the extern "C" surface of include/frostgpu.h.
//
// There is deliberately no CPU execution path in this file: without a CUDA device fgpu_init fails
// with FGPU_ERR_NO_DEVICE and nothing else can run.
#include <cuda_runtime.h>
#include <unistd.h>

#include <algorithm>
#include <array>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <limits>
#include <map>
#include <memory>
#include <mutex>
#include <new>
#include <set>
#include <sstream>
#include <string>
#include <vector>

#include "../../include/frostgpu.h"
#include "arrow_export.h"
#include "context.h"
#include "device_types.h"
#include "kernels.h"
#include "part_store.h"
#include "residency.h"
#include "result.h"

using namespace fgpu;

namespace {

struct ExprNode {
  int32_t kind = 0, op = 0, left = -1, right = -1;
  std::string name;
  int32_t lit_type = FGPU_SCALAR_NULL;
  int64_t lit_i = 0;
  double lit_f = 0;
  std::string lit_bytes;
  fgpu_match_fn match = nullptr;
  void* match_user = nullptr;
};

const char* op_string(int op) {  // logicalplan.Op.String(), expr.go:35-72
  switch (op) {
    case FGPU_OP_EQ: return "==";
    case FGPU_OP_NOT_EQ: return "!=";
    case FGPU_OP_LT: return "<";
    case FGPU_OP_LT_EQ: return "<=";
    case FGPU_OP_GT: return ">";
    case FGPU_OP_GT_EQ: return ">=";
    case FGPU_OP_REGEX_MATCH: return "=~";
    case FGPU_OP_REGEX_NOT_MATCH: return "!~";
    case FGPU_OP_AND: return "&&";
    case FGPU_OP_OR: return "||";
    case FGPU_OP_ADD: return "+";
    case FGPU_OP_SUB: return "-";
    case FGPU_OP_MUL: return "*";
    case FGPU_OP_DIV: return "/";
    case FGPU_OP_CONTAINS: return "contains";
    case FGPU_OP_NOT_CONTAINS: return "not contains";
    default: return "?";
  }
}

const char* agg_string(int f) {  // logicalplan.AggFunc.String(), expr.go:731-750
  switch (f) {
    case FGPU_AGG_SUM: return "sum";
    case FGPU_AGG_MIN: return "min";
    case FGPU_AGG_MAX: return "max";
    case FGPU_AGG_COUNT: return "count";
    case FGPU_AGG_AVG: return "avg";
    case FGPU_AGG_UNIQUE: return "unique";
    default: return "?";
  }
}

}  // namespace

// Mailbox communicator of one rank (see comm.cu).
struct CommHandle {  // what travels between the ranks (FGPU_COMM_HANDLE_BYTES)
  uint32_t magic;
  int32_t device;
  uint64_t pid, ptr, total, slot_bytes;
  int32_t n, rank;
  cudaIpcMemHandle_t ipc;
};
static_assert(sizeof(CommHandle) <= FGPU_COMM_HANDLE_BYTES, "handle fits its blob");
constexpr uint32_t kCommMagic = 0x46474d42u;  // "FGMB"

// The FROSTGPU_* development switches (tests and measurements use them to force a kernel or a layout), parsed.  A
// NO_* switch, TA_GLOBAL, TA_CARRY and PROFILE are on when they are set at all.  `key` lists every switch that is set
// (NAME=value;): a compiled plan is only reused under the key it was compiled with.
struct Switches {
  bool no_tile = false, no_runs = false, no_prune = false, no_fast = false, no_fuse = false, no_take = false, no_prefix = false;
  bool no_exec_cache = false, no_plan_cache = false, profile = false;  // profile: host phase times of every Execute on stderr
  bool ta_global = false, ta_carry = false;      // tile kernel: table in global memory; never the carry-free 32-bit Sums
  int ta_tile = 0, ta_stages = 0, ta_chunk = 0;  // tile kernel: forced tile rows, ring depth, tiles per CTA turn (0: chosen)
  int vl = 256, ring = 3;                        // scan kernel: rows per warp vector, ring depth
  int rt_tile = 4096, rt_stages = 0, rt_span = 0, rt_warps = 0;  // sorted-run kernel: tile rows, forced layout (0: chosen)
  std::string key;
};

Switches read_switches() {
  Switches w;
  auto get = [&w](const char* name) {  // every switch read lands in the key
    const char* v = getenv(name);
    if (v) { w.key += name; w.key += '='; w.key += v; w.key += ';'; }
    return v;
  };
  auto num = [&get](const char* name, int d) { const char* v = get(name); return v ? atoi(v) : d; };
  static const std::pair<const char*, bool Switches::*> kFlags[] = {
      {"FROSTGPU_NO_TILE", &Switches::no_tile},     {"FROSTGPU_NO_RUNS", &Switches::no_runs},     {"FROSTGPU_NO_PRUNE", &Switches::no_prune},
      {"FROSTGPU_NO_FAST", &Switches::no_fast},     {"FROSTGPU_NO_FUSE", &Switches::no_fuse},     {"FROSTGPU_NO_TAKE", &Switches::no_take},
      {"FROSTGPU_NO_PREFIX", &Switches::no_prefix}, {"FROSTGPU_TA_GLOBAL", &Switches::ta_global}, {"FROSTGPU_TA_CARRY", &Switches::ta_carry},
      {"FROSTGPU_NO_EXEC_CACHE", &Switches::no_exec_cache}, {"FROSTGPU_NO_PLAN_CACHE", &Switches::no_plan_cache}, {"FROSTGPU_PROFILE", &Switches::profile}};
  for (const auto& f : kFlags) w.*f.second = get(f.first) != nullptr;
  w.ta_tile = num("FROSTGPU_TA_TILE", 0);
  w.ta_stages = num("FROSTGPU_TA_STAGES", 0);
  if (const char* v = get("FROSTGPU_TA_CHUNK")) w.ta_chunk = std::max(1, atoi(v));
  w.vl = num("FROSTGPU_VL", 256);
  if (w.vl != 128 && w.vl != 256 && w.vl != 512 && w.vl != 1024) w.vl = 512;
  w.ring = std::min(4, std::max(2, num("FROSTGPU_RING", 3)));
  const int rt = num("FROSTGPU_RT_TILE", 0);
  if (rt == 1024 || rt == 2048 || rt == 4096 || rt == 8192) w.rt_tile = rt;
  w.rt_stages = num("FROSTGPU_RT_STAGES", 0);
  w.rt_span = num("FROSTGPU_RT_SPAN", 0);
  w.rt_warps = num("FROSTGPU_RT_WARPS", 0);
  return w;
}

extern "C" char** environ;
// Called per Execute: the environment is only parsed again when its block looks changed (same array, same entry
// pointers: setenv / putenv replace an entry).
Switches switches() {
  static std::mutex mu;
  static Switches cached;
  static uint64_t cached_sig = 0;
  uint64_t sig = 0x9e3779b97f4a7c15ull ^ uint64_t(reinterpret_cast<uintptr_t>(environ));
  for (char** e = environ; e && *e; e++) sig = (sig ^ uint64_t(reinterpret_cast<uintptr_t>(*e))) * 0x100000001b3ull;
  std::lock_guard<std::mutex> lk(mu);
  if (sig != cached_sig || cached_sig == 0) {
    cached = read_switches();
    cached_sig = sig;
  }
  return cached;
}

struct PhaseClock {
  bool on = switches().profile;
  std::chrono::steady_clock::time_point t0 = std::chrono::steady_clock::now();
  std::string line;
  void mark(const char* what) {
    if (!on) return;
    auto t = std::chrono::steady_clock::now();
    char buf[96];
    snprintf(buf, sizeof buf, " %s=%.0fus", what, std::chrono::duration<double, std::micro>(t - t0).count());
    line += buf;
    t0 = t;
  }
  void flush(const char* tag) {
    if (on && !line.empty()) fprintf(stderr, "[frostgpu %s]%s\n", tag, line.c_str());
    line.clear();
  }
};

// A prepared plan.  Prepared queries with the same plan text share ONE of these through the context's plan table,
// so that the shim's prepare-per-Execute still reuses the compiled plan and its device state.
struct QueryPlan {
  // the compiled plan of the last Execute, reused while the table (its parts, its dictionaries) and the read
  // transaction are the same: a prepared query re-executed on an unchanged table skips plan compilation
  mutable std::shared_ptr<void> plan_cache;  // Compiled
  mutable uint64_t cache_epoch = 0, cache_tx = 0;
  mutable std::string cache_env;  // the FROSTGPU_* development switches the plan was compiled under
  fgpu_ctx* ctx = nullptr;
  std::string table;
  int32_t kind = 0;
  std::vector<ExprNode> exprs;
  int32_t filter = -1;
  std::vector<int32_t> group_by;
  std::vector<fgpu_agg> aggs;

  std::string expr_name(int i) const {  // Expr.Name(), expr.go:181,326,568,623
    const ExprNode& e = exprs[size_t(i)];
    switch (e.kind) {
      case FGPU_EXPR_COLUMN:
      case FGPU_EXPR_DYNCOLUMN: return e.name;
      case FGPU_EXPR_LITERAL: {
        if (e.lit_type == FGPU_SCALAR_INT64) return std::to_string(e.lit_i);
        if (e.lit_type == FGPU_SCALAR_FLOAT64) {
          char buf[64];
          snprintf(buf, sizeof buf, "%g", e.lit_f);
          return buf;
        }
        if (e.lit_type == FGPU_SCALAR_STRING) return e.lit_bytes;
        return "null";
      }
      case FGPU_EXPR_BINARY: return expr_name(e.left) + " " + op_string(e.op) + " " + expr_name(e.right);
    }
    return "?";
  }
};

struct fgpu_query {
  fgpu_ctx* ctx = nullptr;
  std::shared_ptr<QueryPlan> plan;
};

struct fgpu_result {
  fgpu_ctx* ctx = nullptr;
  fgpu_stats stats{};
  // compiled state kept for partial/merge
  QueryDesc qd{};
  FinalizeDesc fd{};
  DevBuf table, aux, cnt;
  DevBuf segs;  // the prefix path's segment table (see ExecCache::segs) when the plan is not cached
  size_t table_bytes = 0;
  unsigned int* cnt_ptr = nullptr;  // group counter inside `aux` when the scan counted the result rows
  bool groups_known = false;  // the scan's own stream already counted the result rows
  unsigned int n_groups = 0;
  ResultShape shape;
  // finished records
  std::vector<std::vector<OwnedColumn>> records;
  std::vector<int64_t> record_rows;
  size_t next = 0;
  bool finalized = false;
  // The finished result: an empty one has no record (finishAggregate, aggregate.go:547-549; filter.go:264-266).
  void finish(std::vector<OwnedColumn>&& cols, size_t rows) {
    if (rows > 0) {
      records.push_back(std::move(cols));
      record_rows.push_back(int64_t(rows));
    }
    finalized = true;
  }
  bool rows_plan = false;
  bool rows_no_nulls = false;  // rows plan produced by the take kernels: no projected value is NULL
  // collective Execute between its two halves: the partial table is pushed, the merge is still to come
  bool pending = false;
  void* pending_cached = nullptr;              // ExecCache: the plan-owned device state holds the table (else `table`)
  std::shared_ptr<void> plan_keep;             // keeps that plan alive
  uint64_t pending_seq = 0, pending_bytes = 0;
};

namespace {

struct VisibleRG {
  Part* part;
  RowGroupHost* rg;
  uint64_t skip_slots = 0;               // bit s: slot s is not read in this row group (its leaf is decided by statistics)
  uint8_t leaf_mode[kMaxLeaves] = {0};   // LeafMode per leaf decided from the chunk statistics (LM_EVAL: undecided)
  uint8_t key_leaf_mode[kMaxLeaves] = {0};  // the same for the boolean keys' leaves (never drops the row group)
};


// One predicate leaf on the host.
struct LeafHost {
  std::string column;
  int slot = -1;  // -1: column absent from every visible row group
  int op = 0;
  const ExprNode* lit = nullptr;
  const ExprNode* bin = nullptr;
  size_t lut_off = size_t(-1);  // dictionary leaves: offset of the per-global-id result bytes in the LUT blob
  // numeric leaves, canonical form (see LeafDesc)
  bool numeric = false, never = false, neg = false, cmp_float = false, null_literal = false;
  int64_t lo_i = 0, hi_i = 0;
  double lo_f = 0, hi_f = 0;
  uint8_t missing_mode = LM_ALL;  // behaviour on row groups that lack the column
};

bool bytes_contains(const std::string& hay, const std::string& needle) {
  if (needle.empty()) return true;
  return hay.find(needle) != std::string::npos;
}

// Missing-column rules, binaryscalarexpr.go:47-73 and regexpfilter.go:23-33.  Returns LM_ALL / LM_NONE.
uint8_t missing_column_mode(const LeafHost& l) {
  const ExprNode& lit = *l.lit;
  switch (l.op) {
    case FGPU_OP_EQ:
      if (lit.lit_type == FGPU_SCALAR_STRING && !lit.lit_bytes.empty()) return LM_NONE;
      return LM_ALL;
    case FGPU_OP_NOT_EQ:
      if (lit.lit_type == FGPU_SCALAR_NULL) return LM_NONE;
      return LM_ALL;
    case FGPU_OP_LT: case FGPU_OP_LT_EQ: case FGPU_OP_GT: case FGPU_OP_GT_EQ:
      return LM_NONE;
    case FGPU_OP_REGEX_MATCH:
    case FGPU_OP_REGEX_NOT_MATCH: {
      bool empty_match = l.bin->match ? l.bin->match(l.bin->match_user, reinterpret_cast<const uint8_t*>(""), 0) != 0 : false;
      bool not_match = l.op == FGPU_OP_REGEX_NOT_MATCH;
      return ((not_match && !empty_match) || (!not_match && empty_match)) ? LM_ALL : LM_NONE;
    }
    default:
      return LM_ALL;  // contains / not contains fall through to "all rows" (:71)
  }
}

// Result of a dictionary leaf for one dictionary value (non-NULL row).
bool dict_leaf_value(const LeafHost& l, const std::string& v) {
  const ExprNode& lit = *l.lit;
  switch (l.op) {
    case FGPU_OP_EQ: return lit.lit_type != FGPU_SCALAR_NULL && v == lit.lit_bytes;
    case FGPU_OP_NOT_EQ: return lit.lit_type == FGPU_SCALAR_NULL ? true : v != lit.lit_bytes;
    case FGPU_OP_CONTAINS:
      return lit.lit_type == FGPU_SCALAR_NULL ? true : bytes_contains(v, lit.lit_bytes);
    case FGPU_OP_NOT_CONTAINS:
      return lit.lit_type == FGPU_SCALAR_NULL ? true : !bytes_contains(v, lit.lit_bytes);
    case FGPU_OP_REGEX_MATCH:
      return l.bin->match(l.bin->match_user, reinterpret_cast<const uint8_t*>(v.data()), v.size()) != 0;
    case FGPU_OP_REGEX_NOT_MATCH:
      return l.bin->match(l.bin->match_user, reinterpret_cast<const uint8_t*>(v.data()), v.size()) == 0;
  }
  return false;
}

// "column op literal" on an int64 column as an inclusive range, optionally negated (see LeafDesc).
void canonical_int_range(int op, int64_t v, int64_t* lo, int64_t* hi, bool* neg) {
  const int64_t kMin = std::numeric_limits<int64_t>::min(), kMax = std::numeric_limits<int64_t>::max();
  *lo = kMax; *hi = kMin;  // empty
  *neg = false;
  switch (op) {
    case FGPU_OP_EQ: *lo = *hi = v; break;
    case FGPU_OP_NOT_EQ: *lo = *hi = v; *neg = true; break;
    case FGPU_OP_LT: if (v != kMin) { *lo = kMin; *hi = v - 1; } break;
    case FGPU_OP_LT_EQ: *lo = kMin; *hi = v; break;
    case FGPU_OP_GT: if (v != kMax) { *lo = v + 1; *hi = kMax; } break;
    default: *lo = v; *hi = kMax; break;
  }
}

// "column op literal" compared as float64, as an inclusive range, optionally negated (see LeafDesc).  A NaN literal
// gives the empty range: x != NaN holds for every non-NULL x, every other comparison with NaN for none.
void canonical_float_range(int op, double v, double* lo, double* hi, bool* neg) {
  const double kInf = std::numeric_limits<double>::infinity();
  *lo = kInf; *hi = -kInf;  // empty
  *neg = op == FGPU_OP_NOT_EQ;
  if (std::isnan(v)) return;
  switch (op) {
    case FGPU_OP_EQ: case FGPU_OP_NOT_EQ: *lo = *hi = v; break;
    case FGPU_OP_LT: if (v != -kInf) { *lo = -kInf; *hi = std::nextafter(v, -kInf); } break;
    case FGPU_OP_LT_EQ: *lo = -kInf; *hi = v; break;
    case FGPU_OP_GT: if (v != kInf) { *lo = std::nextafter(v, kInf); *hi = kInf; } break;
    default: *lo = v; *hi = kInf; break;
  }
}

// What the chunk statistics [mn, mx] (bounds of the non-null values) decide about an int64 range leaf for a
// whole row group: LM_NONE no row can pass, LM_ALL every row passes (needs a chunk without NULLs), LM_EVAL
// undecided.  The row-group filter of the reference (expr/binaryscalarexpr.go:84-190) answers the first question.
uint8_t stats_leaf_mode(int64_t lo, int64_t hi, bool neg, int64_t mn, int64_t mx, bool no_nulls) {
  const bool disjoint = mx < lo || mn > hi;
  const bool inside = mn >= lo && mx <= hi;
  if (!neg) return disjoint ? LM_NONE : ((inside && no_nulls) ? LM_ALL : LM_EVAL);
  return inside ? LM_NONE : ((disjoint && no_nulls) ? LM_ALL : LM_EVAL);
}

// The decision leaf_mode() takes for an int64 range leaf on one chunk, also behind the host-only test hook
// fgpu_rowgroup_leaf_mode: an all-NULL chunk has no usable bounds (nothing is decided from statistics).
uint8_t chunk_leaf_mode(int64_t lo, int64_t hi, bool neg, bool has_bounds, int64_t mn, int64_t mx, int64_t null_count, int64_t num_values) {
  if (!has_bounds || (null_count >= 0 && null_count == num_values)) return LM_EVAL;
  return stats_leaf_mode(lo, hi, neg, mn, mx, null_count == 0);
}

// The launches of an aggregate scan before the general k_scan, in issue order: k_runs_prefix when the plan has prefix
// row groups (it stores every slot of the table), k_table_init otherwise, then sorted runs (k_runs_tma) and tile
// aggregate (k_tile_agg), which add to the table atomically.
struct ScanLaunch {
  bool runs = false, prefix = false, tile = false;
  RunsDesc rd{};
  int runs_nl = 0, runs_nk = 0, runs_na = 0;
  PrefixDesc pd{};
  TileAggDesc td{};
};

// Device and page-locked state of a compiled plan that every Execute of a prepared query reuses while the plan is
// valid (same table epoch, same read transaction): the descriptor block is uploaded once, the aggregate table and
// its counters are one persistent allocation, and the table comes back to page-locked memory with ONE copy and ONE
// stream synchronisation per Execute; dense tables of this size are compacted into the result record on the host.
struct ExecCache {
  DevBuf aux, table, out;         // descriptors; [aggregate table | counters 128 B]; compacted result image
  // The prefix path's segment table (seg_off, seg: PrefixBuildDesc), built by the plan's first Execute.  It holds only
  // dense slots and row positions derived from the key columns' run directories, never a value: every Execute reads
  // the Sum inputs' prefix images afresh and stores every slot, so no aggregate survives from one Execute to the next.
  DevBuf segs;
  DenseOut dout{};
  size_t out_bytes = 0;
  std::vector<std::unique_ptr<OwnedColumn>> dict_template;  // per key: the whole dictionary, ready to copy (small dictionaries)
  PinnedBlock pinned;             // host image of the compacted result (from the context's page-locked pool)
  size_t table_bytes = 0;
  bool ready = false;
  QueryDesc qd{};
  const QueryDesc* qdesc_dev = nullptr;
  ScanLaunch launch;
  fgpu_stats stats{};             // everything about the scan that does not change between Executes
  ResultShape shape;
};

struct Compiled {
  std::unique_ptr<ExecCache> exec;
  std::vector<VisibleRG> rgs;
  std::vector<std::string> slot_names;
  std::vector<uint8_t> slot_types;
  std::vector<uint8_t> slot_needed;  // 0: only named by Count(), whose result does not depend on the values
  std::vector<LeafHost> leaves;
  std::vector<uint8_t> filter_prog;
  // boolean Distinct keys: their leaves and postfix programs, apart from the filter's (see BoolKeys)
  std::vector<LeafHost> key_leaves;
  std::vector<uint8_t> key_prog;
  size_t filter_leaves = 0;  // the filter's leaves as written, before fuse_conjunction: the keys' share of kMaxLeaves
  BoolKeys bool_keys{};
  std::vector<KeyOut> keys;
  std::vector<int> key_slots;
  QueryDesc qd{};
  std::vector<uint32_t> dense_radix;
  uint64_t total_rows = 0;
  uint64_t group_bound = 0;
  uint64_t h2d_bytes = 0;  // column uploads this query triggered
  uint32_t pruned_row_groups = 0;
  uint64_t touched_rows = ~uint64_t(0);  // rows of the row groups that survive pruning (~0: nothing was pruned)
  uint32_t radix(int k) const { return dense_radix[size_t(k)] ? dense_radix[size_t(k)] : 1; }  // (int64 keys have none)
  bool has_bool_keys() const { return !key_leaves.empty(); }  // (every boolean key has a leaf)
  bool has_unique() const {  // a Unique aggregate: only k_scan's general path feeds its cells the NULL rows
    for (int a = 0; a < qd.n_aggs; a++)
      if (qd.aggs[a].unique) return true;
    return false;
  }
};

// A boolean expression -> postfix program over its leaves, appended to *leaves and *prog.  `other`: leaves of the plan
// kept elsewhere, which share the kMaxLeaves budget (the filter's, when a boolean key is compiled).
int32_t compile_filter(const QueryPlan& q, int node, std::vector<LeafHost>* leaves, std::vector<uint8_t>* prog,
                       const std::map<std::string, int>& slot_of, size_t other = 0) {
  const ExprNode& e = q.exprs[size_t(node)];
  if (e.kind != FGPU_EXPR_BINARY) return fail(FGPU_ERR_UNSUPPORTED, "unsupported boolean expression");
  if (e.op == FGPU_OP_AND || e.op == FGPU_OP_OR) {
    int32_t rc = compile_filter(q, e.left, leaves, prog, slot_of, other);
    if (rc) return rc;
    rc = compile_filter(q, e.right, leaves, prog, slot_of, other);
    if (rc) return rc;
    prog->push_back(e.op == FGPU_OP_AND ? 0x80 : 0x81);
    return FGPU_OK;
  }
  switch (e.op) {
    case FGPU_OP_EQ: case FGPU_OP_NOT_EQ: case FGPU_OP_LT: case FGPU_OP_LT_EQ: case FGPU_OP_GT: case FGPU_OP_GT_EQ:
    case FGPU_OP_REGEX_MATCH: case FGPU_OP_REGEX_NOT_MATCH: case FGPU_OP_CONTAINS: case FGPU_OP_NOT_CONTAINS:
      break;
    default:
      return fail(FGPU_ERR_UNSUPPORTED, std::string("unsupported filter operator ") + op_string(e.op));
  }
  const ExprNode& l = q.exprs[size_t(e.left)];
  const ExprNode& r = q.exprs[size_t(e.right)];
  if (l.kind != FGPU_EXPR_COLUMN) return fail(FGPU_ERR_INVALID, "left side of binary expression must be a column");
  if (r.kind != FGPU_EXPR_LITERAL) return fail(FGPU_ERR_INVALID, "right side of binary expression must be a literal");
  if ((e.op == FGPU_OP_REGEX_MATCH || e.op == FGPU_OP_REGEX_NOT_MATCH) && !e.match)
    return fail(FGPU_ERR_INVALID, "regex leaf without a matcher");
  if (leaves->size() + other >= size_t(kMaxLeaves)) return fail(FGPU_ERR_UNSUPPORTED, "too many predicate leaves");
  LeafHost lh;
  lh.column = l.name;
  lh.op = e.op;
  lh.lit = &r;
  lh.bin = &e;
  auto it = slot_of.find(l.name);
  lh.slot = (it == slot_of.end()) ? -1 : it->second;
  prog->push_back(uint8_t(leaves->size()));
  leaves->push_back(std::move(lh));
  return FGPU_OK;
}

int32_t compile_agg_expr(const QueryPlan& q, int node, const std::map<std::string, int>& slot_of, const Compiled& c,
                         std::vector<ProgOp>* prog, bool* any_float, bool* any_int_col) {
  const ExprNode& e = q.exprs[size_t(node)];
  if (e.kind == FGPU_EXPR_COLUMN) {
    auto it = slot_of.find(e.name);
    if (it == slot_of.end()) return fail(FGPU_ERR_NOT_FOUND, "aggregate field(s) not found [\"" + e.name + "\"], aggregations are not possible without it");
    uint8_t t = c.slot_types[size_t(it->second)];
    if (t == ST_DICT) return fail(FGPU_ERR_UNSUPPORTED, "aggregation over a non-numeric column: " + e.name);
    if (t == ST_F64) *any_float = true; else *any_int_col = true;
    ProgOp op{};
    op.op = PO_LOAD;
    op.slot = uint8_t(it->second);
    prog->push_back(op);
    return FGPU_OK;
  }
  if (e.kind == FGPU_EXPR_LITERAL) {
    ProgOp op{};
    op.op = PO_CONST;
    if (e.lit_type == FGPU_SCALAR_INT64) op.imm = e.lit_i;
    else if (e.lit_type == FGPU_SCALAR_FLOAT64) { std::memcpy(&op.imm, &e.lit_f, 8); op.slot = 1; *any_float = true; }
    else return fail(FGPU_ERR_UNSUPPORTED, "non-numeric literal in arithmetic expression");
    prog->push_back(op);
    return FGPU_OK;
  }
  if (e.kind == FGPU_EXPR_BINARY && e.op >= FGPU_OP_ADD && e.op <= FGPU_OP_DIV) {
    int32_t rc = compile_agg_expr(q, e.left, slot_of, c, prog, any_float, any_int_col);
    if (rc) return rc;
    rc = compile_agg_expr(q, e.right, slot_of, c, prog, any_float, any_int_col);
    if (rc) return rc;
    ProgOp op{};
    op.op = uint8_t(PO_ADD + (e.op - FGPU_OP_ADD));
    prog->push_back(op);
    return FGPU_OK;
  }
  return fail(FGPU_ERR_UNSUPPORTED, "unsupported aggregate expression");
}

void collect_columns(const QueryPlan& q, int node, std::vector<std::string>* out) {
  if (node < 0) return;
  const ExprNode& e = q.exprs[size_t(node)];
  if (e.kind == FGPU_EXPR_COLUMN) out->push_back(e.name);
  if (e.kind == FGPU_EXPR_BINARY) {
    collect_columns(q, e.left, out);
    collect_columns(q, e.right, out);
  }
}

// The row-group filter LSM.Scan applies to the row groups of Parquet parts before they reach the plan
// (index/lsm.go:437; expr/filter.go:208-268 builds And / Or / BinaryScalarExpr, everything else is AlwaysTrue;
// expr/binaryscalarexpr.go:42-190 answers "may this chunk hold a matching value" from the null count and the
// bounds).  Its rules for a column that is MISSING from the row group (:47-73) differ from the physical plan's
// (physicalplan/binaryscalarexpr.go:47-73): `missing == 5`, `missing != 5`, `missing != ""` and every ordering
// comparison drop the row group here, so its rows never reach the plan.
int stat_compare(const ChunkHost& ch, bool use_max, const ExprNode& lit, bool* ok) {
  *ok = false;
  if (ch.phys == PT_INT64 && lit.lit_type == FGPU_SCALAR_INT64 && ch.has_minmax) {
    const int64_t v = use_max ? ch.max_bits : ch.min_bits;
    *ok = true;
    return v < lit.lit_i ? -1 : (v > lit.lit_i ? 1 : 0);
  }
  if (ch.phys == PT_DOUBLE && lit.lit_type == FGPU_SCALAR_FLOAT64 && ch.has_minmax) {
    double v;
    std::memcpy(&v, use_max ? &ch.max_bits : &ch.min_bits, 8);
    *ok = true;
    return v < lit.lit_f ? -1 : (v > lit.lit_f ? 1 : 0);
  }
  if (ch.phys == PT_BYTE_ARRAY && lit.lit_type == FGPU_SCALAR_STRING && ch.has_minmax_str) {
    const std::string& v = use_max ? ch.max_str : ch.min_str;
    *ok = true;
    const int c = v.compare(lit.lit_bytes);
    return c < 0 ? -1 : (c > 0 ? 1 : 0);
  }
  return 0;
}

// Split-block bloom filter of the chunk against a non-null literal (expr/binaryscalarexpr.go:104-118: parquet-go hashes
// the PLAIN encoding of the value with XXH64): false = the value is definitely not in the chunk.  Chunks without a
// filter, and literals whose type does not match the column's, answer true.
bool bloom_may_contain(const ChunkHost& ch, const ExprNode& lit) {
  if (ch.bloom.empty()) return true;
  uint64_t h;
  if (ch.phys == PT_INT64 && lit.lit_type == FGPU_SCALAR_INT64) {
    uint8_t b[8];
    std::memcpy(b, &lit.lit_i, 8);
    h = xxhash64(b, 8, 0);
  } else if (ch.phys == PT_DOUBLE && lit.lit_type == FGPU_SCALAR_FLOAT64) {
    uint8_t b[8];
    std::memcpy(b, &lit.lit_f, 8);
    h = xxhash64(b, 8, 0);
  } else if (ch.phys == PT_BYTE_ARRAY && lit.lit_type == FGPU_SCALAR_STRING) {
    h = xxhash64(reinterpret_cast<const uint8_t*>(lit.lit_bytes.data()), lit.lit_bytes.size(), 0);
  } else {
    return true;
  }
  return sbbf_check(ch.bloom.data(), uint32_t(ch.bloom.size()), h);
}

bool rg_may_match(const QueryPlan& q, int node, const RowGroupHost& rg) {
  if (node < 0) return true;
  const ExprNode& e = q.exprs[size_t(node)];
  if (e.kind != FGPU_EXPR_BINARY) return true;
  if (e.op == FGPU_OP_AND) return rg_may_match(q, e.left, rg) && rg_may_match(q, e.right, rg);
  if (e.op == FGPU_OP_OR) return rg_may_match(q, e.left, rg) || rg_may_match(q, e.right, rg);
  if (e.op < FGPU_OP_EQ || e.op > FGPU_OP_GT_EQ) return true;  // AlwaysTrueFilter
  const ExprNode& l = q.exprs[size_t(e.left)];
  const ExprNode& lit = q.exprs[size_t(e.right)];
  if (l.kind != FGPU_EXPR_COLUMN || lit.kind != FGPU_EXPR_LITERAL) return true;
  auto it = rg.cols.find(l.name);
  if (it == rg.cols.end()) {  // :47-73
    if (lit.lit_type == FGPU_SCALAR_NULL) {
      if (e.op == FGPU_OP_EQ) return true;
      if (e.op == FGPU_OP_NOT_EQ) return false;
    }
    if (lit.lit_type == FGPU_SCALAR_STRING) {
      if (e.op == FGPU_OP_EQ && lit.lit_bytes.empty()) return true;
      if (e.op == FGPU_OP_NOT_EQ && !lit.lit_bytes.empty()) return true;
    }
    return false;
  }
  const ChunkHost& ch = it->second;
  const int64_t nulls = ch.null_count;  // -1: not recorded
  const bool full_of_nulls = nulls >= 0 && uint64_t(nulls) == rg.n_rows;
  bool ok;
  if (e.op == FGPU_OP_EQ) {
    if (lit.lit_type == FGPU_SCALAR_NULL) return nulls != 0;
    if (full_of_nulls) return false;
    // the reference asks the bloom filter when the chunk has one and the bounds otherwise (:104-118); both are true
    // negatives, so both are asked here
    if (!bloom_may_contain(ch, lit)) return false;
    const int cmax = stat_compare(ch, true, lit, &ok);
    if (!ok) return true;
    const int cmin = stat_compare(ch, false, lit, &ok);
    if (!ok) return true;
    return cmax >= 0 && cmin <= 0;
  }
  if (lit.lit_type == FGPU_SCALAR_NULL) return true;
  if (full_of_nulls) return false;
  switch (e.op) {
    case FGPU_OP_LT_EQ: { const int c = stat_compare(ch, false, lit, &ok); return !ok || c <= 0; }
    case FGPU_OP_LT: { const int c = stat_compare(ch, false, lit, &ok); return !ok || c < 0; }
    case FGPU_OP_GT: { const int c = stat_compare(ch, true, lit, &ok); return !ok || c > 0; }
    case FGPU_OP_GT_EQ: { const int c = stat_compare(ch, true, lit, &ok); return !ok || c >= 0; }
    default: return true;  // != : left to the execution engine
  }
}

// The plan's columns resolved against the visible row groups.
struct Columns {
  std::map<std::string, int> slot_of;
  std::vector<std::string> key_names;       // group-by / distinct / projected columns and computed keys, in plan order
  std::map<std::string, int32_t> key_expr;  // computed keys: name -> expression node
  std::map<std::string, int32_t> bool_key;  // boolean Distinct keys (value > 0): name -> expression node

  // 1 for the slot of each column whose values the plan reads: keys, computed-key and aggregate inputs and,
  // with_filter, the filter's.  Count(col) counts rows, NULLs included (aggregate.go:929-950): its input column is
  // never read, so it is neither uploaded nor staged unless something else in the query needs it.
  std::vector<uint8_t> value_slots(const QueryPlan& q, bool with_filter) const {
    std::vector<std::string> need = key_names;
    for (auto& kv : key_expr) collect_columns(q, kv.second, &need);
    if (with_filter) collect_columns(q, q.filter, &need);
    for (auto& kv : bool_key)  // read like the filter's: not in a row group where statistics decide every leaf on them
      if (with_filter) collect_columns(q, kv.second, &need);
    for (const fgpu_agg& a : q.aggs)
      if (a.func != FGPU_AGG_COUNT) collect_columns(q, a.expr, &need);
    std::vector<uint8_t> out(slot_of.size(), 0);
    for (auto& n : need) {
      auto it = slot_of.find(n);
      if (it != slot_of.end()) out[size_t(it->second)] = 1;
    }
    return out;
  }
};

// Column types, group keys (a computed key, arithmetic over int64 columns like the sqlparse pre-projection
// `(timestamp / 1000) * 1000 as bucket`, is named after its expression and carries the expression's node) and one
// slot per column the keys, the filter, the aggregates and the computed keys name.
int32_t resolve_columns(const QueryPlan& q, const Table& table, Compiled* c, Columns* k) {
  std::map<std::string, uint8_t> present;  // every column name present in a visible row group, with its type (0xff: unreadable)
  for (const VisibleRG& v : c->rgs) {
    for (auto& kv : v.rg->cols) {
      uint8_t t = kv.second.phys == PT_BYTE_ARRAY ? ST_DICT : (kv.second.phys == PT_DOUBLE ? ST_F64 : ST_I64);
      if (kv.second.phys != PT_BYTE_ARRAY && kv.second.phys != PT_DOUBLE && kv.second.phys != PT_INT64) t = 0xff;
      auto it = present.find(kv.first);
      if (it == present.end()) present.emplace(kv.first, t);
      else if (it->second != t) return fail(FGPU_ERR_UNSUPPORTED, "column " + kv.first + " changes type between parts");
    }
  }
  // string columns whose dictionaries were preloaded (identically on every rank of a multi-GPU run) count
  // as present even when no local row group holds them: the key set, and with it the shape of the partial
  // aggregate table, must not depend on which parts a rank happens to own
  for (auto& kv : table.dicts)
    if (kv.second.preloaded && !present.count(kv.first)) present.emplace(kv.first, uint8_t(ST_DICT));
  std::vector<std::string>& key_names = k->key_names;
  auto add_key_name = [&](const std::string& name) {  // first occurrence only
    if (std::find(key_names.begin(), key_names.end(), name) == key_names.end()) key_names.push_back(name);
  };
  for (int32_t g : q.group_by) {
    const ExprNode& e = q.exprs[size_t(g)];
    if (e.kind == FGPU_EXPR_COLUMN) {
      if (present.count(e.name)) add_key_name(e.name);
    } else if (e.kind == FGPU_EXPR_DYNCOLUMN) {
      std::string prefix = e.name + ".";  // DynamicColumn.MatchColumn, expr.go:564
      for (auto& kv : present)
        if (kv.first.compare(0, prefix.size(), prefix) == 0) add_key_name(kv.first);
    } else if (e.kind == FGPU_EXPR_BINARY && e.op >= FGPU_OP_ADD && e.op <= FGPU_OP_DIV && q.kind == FGPU_PLAN_AGGREGATE) {
      const std::string name = q.expr_name(g);
      if (present.count(name)) return fail(FGPU_ERR_UNSUPPORTED, "computed group key shadows a column: " + name);
      add_key_name(name);
      k->key_expr[name] = g;
    } else if (e.kind == FGPU_EXPR_BINARY && q.kind == FGPU_PLAN_DISTINCT &&
               ((e.op >= FGPU_OP_EQ && e.op <= FGPU_OP_GT_EQ) || e.op == FGPU_OP_REGEX_MATCH || e.op == FGPU_OP_REGEX_NOT_MATCH ||
                e.op == FGPU_OP_AND || e.op == FGPU_OP_OR || e.op == FGPU_OP_CONTAINS || e.op == FGPU_OP_NOT_CONTAINS)) {
      // boolean key: Builder.Distinct projects its expressions first (builder.go:117-134), a comparison as the filter's
      // bitmap (boolExprProjection, project.go:397-467).  Present whatever the parts hold, so the key set and the
      // partial-table shape of a multi-rank run do not depend on them.
      const std::string name = q.expr_name(g);
      if (present.count(name)) return fail(FGPU_ERR_UNSUPPORTED, "boolean key shadows a column: " + name);
      add_key_name(name);
      k->bool_key[name] = g;
    } else {
      return fail(FGPU_ERR_UNSUPPORTED, "this group-by expression is not supported on the GPU path");
    }
  }
  if (key_names.size() > size_t(kMaxKeys)) return fail(FGPU_ERR_UNSUPPORTED, "too many group-by columns");
  // slots: key columns first, then the computed keys', the filter's and the aggregates' input columns
  std::vector<std::string> cols;
  for (auto& n : key_names)
    if (!k->key_expr.count(n) && !k->bool_key.count(n)) cols.push_back(n);
  for (auto& kv : k->key_expr) collect_columns(q, kv.second, &cols);
  collect_columns(q, q.filter, &cols);
  for (auto& kv : k->bool_key) collect_columns(q, kv.second, &cols);
  for (const fgpu_agg& a : q.aggs) collect_columns(q, a.expr, &cols);
  for (auto& name : cols) {
    auto it = present.find(name);
    if (k->slot_of.count(name) || it == present.end()) continue;  // absent everywhere: handled by the callers
    if (it->second == 0xff) return fail(FGPU_ERR_UNSUPPORTED, "column " + name + " has a type the GPU engine does not read");
    if (c->slot_names.size() >= size_t(kMaxSlots)) return fail(FGPU_ERR_UNSUPPORTED, "query touches too many columns");
    k->slot_of[name] = int(c->slot_names.size());
    c->slot_names.push_back(name);
    c->slot_types.push_back(it->second);
  }
  c->qd.n_slots = int32_t(c->slot_names.size());
  for (int s = 0; s < c->qd.n_slots; s++) c->qd.slot_type[s] = c->slot_types[size_t(s)];
  c->slot_needed = q.kind == FGPU_PLAN_AGGREGATE ? k->value_slots(q, true) : std::vector<uint8_t>(c->slot_names.size(), 1);
  return FGPU_OK;
}

// The only writer of the filter program in QueryDesc.  Pure conjunctions / disjunctions of leaves reduce to one mask
// test per row.
void set_filter_prog(Compiled* c) {
  QueryDesc& qd = c->qd;
  qd.n_filter_prog = int32_t(c->filter_prog.size());
  std::memset(qd.filter_prog, 0, sizeof qd.filter_prog);
  std::memcpy(qd.filter_prog, c->filter_prog.data(), c->filter_prog.size());
  bool all_and = true, all_or = true;
  uint32_t mask = 0;
  for (uint8_t op : c->filter_prog) {
    if (op < 0x80) mask |= 1u << op;
    else if (op == 0x80) all_or = false;
    else all_and = false;
  }
  qd.filter_mask = mask;
  qd.filter_kind = all_and ? FK_AND : (all_or ? FK_OR : FK_PROGRAM);
}

// Checks a leaf against its column's type and puts a numeric leaf in canonical form (see LeafDesc).
int32_t canonical_leaf(LeafHost* lh, uint8_t st) {
  const ExprNode& lit = *lh->lit;
  if (st == ST_DICT) {
    switch (lh->op) {
      case FGPU_OP_EQ: case FGPU_OP_NOT_EQ: case FGPU_OP_CONTAINS: case FGPU_OP_NOT_CONTAINS:
        if (lit.lit_type != FGPU_SCALAR_NULL && lit.lit_type != FGPU_SCALAR_STRING)
          return fail(FGPU_ERR_UNSUPPORTED, "dictionary column compared with a non-string literal");
        return FGPU_OK;
      case FGPU_OP_REGEX_MATCH: case FGPU_OP_REGEX_NOT_MATCH:
        return FGPU_OK;
      default:  // binaryscalarexpr.go:100-108
        return fail(FGPU_ERR_INVALID, std::string("unsupported operator: ") + op_string(lh->op));
    }
  }
  if (lh->op < FGPU_OP_EQ || lh->op > FGPU_OP_GT_EQ)
    return fail(FGPU_ERR_UNSUPPORTED, std::string("operator ") + op_string(lh->op) + " on a numeric column");
  if (lit.lit_type == FGPU_SCALAR_STRING) return fail(FGPU_ERR_UNSUPPORTED, "numeric column compared with a string literal");
  lh->numeric = true;
  lh->null_literal = lit.lit_type == FGPU_SCALAR_NULL;  // arrow compute against NULL: nothing selected (:143-150)
  lh->cmp_float = (st == ST_F64) || lit.lit_type == FGPU_SCALAR_FLOAT64;
  if (lh->cmp_float) canonical_float_range(lh->op, lit.lit_type == FGPU_SCALAR_FLOAT64 ? lit.lit_f : double(lit.lit_i), &lh->lo_f, &lh->hi_f, &lh->neg);
  else canonical_int_range(lh->op, lit.lit_i, &lh->lo_i, &lh->hi_i, &lh->neg);
  return FGPU_OK;
}

// Conjunction: comparisons on the same numeric column intersect into one range leaf
// (timestamp >= a AND timestamp < b  ->  timestamp in [a, b-1]); a missing column keeps the
// strictest of the merged leaves' missing-column behaviours.
void fuse_conjunction(Compiled* c) {
  std::vector<LeafHost> fused;
  for (LeafHost& lh : c->leaves) {
    bool merged = false;
    if (lh.numeric && !lh.neg && !lh.null_literal && lh.slot >= 0) {
      for (LeafHost& f : fused) {
        if (!f.numeric || f.neg || f.null_literal || f.slot != lh.slot || f.cmp_float != lh.cmp_float) continue;
        if (f.cmp_float) { f.lo_f = std::max(f.lo_f, lh.lo_f); f.hi_f = std::min(f.hi_f, lh.hi_f); }
        else { f.lo_i = std::max(f.lo_i, lh.lo_i); f.hi_i = std::min(f.hi_i, lh.hi_i); }
        if (lh.missing_mode == LM_NONE) f.missing_mode = LM_NONE;
        merged = true;
        break;
      }
    }
    if (!merged) fused.push_back(lh);
  }
  if (fused.size() == c->leaves.size()) return;
  c->leaves.swap(fused);
  c->filter_prog.clear();
  for (size_t l = 0; l < c->leaves.size(); l++) {
    c->filter_prog.push_back(uint8_t(l));
    if (l > 0) c->filter_prog.push_back(0x80);
  }
  set_filter_prog(c);
}

// Stack depth of a postfix program (the kernels keep the stack in 32 bits).
int postfix_depth(const std::vector<uint8_t>& prog, size_t off) {
  int depth = 0, maxd = 0;
  for (size_t i = off; i < prog.size(); i++) {
    if (prog[i] < 0x80) depth++; else depth--;
    maxd = std::max(maxd, depth);
  }
  return maxd;
}

// Missing-column rules and canonical form of every leaf (see LeafHost).
int32_t canonical_leaves(std::vector<LeafHost>* leaves, const std::vector<uint8_t>& slot_types) {
  for (LeafHost& lh : *leaves) {
    lh.missing_mode = missing_column_mode(lh);
    if (lh.slot < 0) continue;
    int32_t rc = canonical_leaf(&lh, slot_types[size_t(lh.slot)]);
    if (rc) return rc;
  }
  return FGPU_OK;
}

LeafDesc leaf_desc(const LeafHost& lh) {
  LeafDesc ld{};
  ld.slot = uint8_t(lh.slot < 0 ? 0xff : lh.slot);
  ld.op = uint8_t(lh.op);
  if (lh.slot < 0) return ld;
  ld.cmp_float = lh.cmp_float;
  ld.neg = lh.neg;
  ld.lo_i = lh.lo_i; ld.hi_i = lh.hi_i;
  ld.lo_f = lh.lo_f; ld.hi_f = lh.hi_f;
  return ld;
}

// The filter: its program, its leaves in canonical form, fused under a conjunction, and their descriptors.
int32_t compile_predicate(const QueryPlan& q, const Switches& w, const std::map<std::string, int>& slot_of, Compiled* c) {
  QueryDesc& qd = c->qd;
  if (q.filter >= 0) {
    int32_t rc = compile_filter(q, q.filter, &c->leaves, &c->filter_prog, slot_of);
    if (rc) return rc;
    if (c->filter_prog.size() > size_t(kMaxFilterProg)) return fail(FGPU_ERR_UNSUPPORTED, "filter expression too large");
    if (postfix_depth(c->filter_prog, 0) > 30) return fail(FGPU_ERR_UNSUPPORTED, "filter expression too deep");
    set_filter_prog(c);
  }
  if (int32_t rc = canonical_leaves(&c->leaves, c->slot_types)) return rc;
  c->filter_leaves = c->leaves.size();
  if (qd.filter_kind == FK_AND && !w.no_fuse) fuse_conjunction(c);
  qd.n_leaves = int32_t(c->leaves.size());
  for (int l = 0; l < qd.n_leaves; l++) {
    const LeafHost& lh = c->leaves[size_t(l)];
    qd.leaves[l] = leaf_desc(lh);
    if (lh.slot >= 0) qd.slot_used_by_leaf[lh.slot] = 1;
  }
  return FGPU_OK;
}

// Boolean Distinct keys: each expression is compiled exactly as a filter would be (same leaves, refusals and
// missing-column rules), into the key leaves and one postfix program per key.  Their leaves share the filter's
// kMaxLeaves budget, counted with the filter's leaves as written (before fusion), so that FROSTGPU_NO_FUSE accepts and
// refuses the same plans; they never take part in the filter's program, its fusion or row-group pruning.
int32_t compile_bool_keys(const QueryPlan& q, const Columns& k, Compiled* c) {
  BoolKeys& bk = c->bool_keys;
  for (size_t i = 0; i < k.key_names.size(); i++) {
    const auto it = k.bool_key.find(k.key_names[i]);
    if (it == k.bool_key.end()) continue;
    const size_t off = c->key_prog.size();
    int32_t rc = compile_filter(q, it->second, &c->key_leaves, &c->key_prog, k.slot_of, c->filter_leaves);
    if (rc) return rc;
    if (c->key_prog.size() > size_t(kMaxFilterProg)) return fail(FGPU_ERR_UNSUPPORTED, "boolean key expressions too large");
    if (postfix_depth(c->key_prog, off) > 30) return fail(FGPU_ERR_UNSUPPORTED, "boolean key expression too deep");
    KeyDesc& kd = c->qd.keys[i];
    kd.is_bool = 1;
    kd.prog_off = uint8_t(off);
    kd.prog_len = uint8_t(c->key_prog.size() - off);
  }
  if (int32_t rc = canonical_leaves(&c->key_leaves, c->slot_types)) return rc;
  bk.n_leaves = int32_t(c->key_leaves.size());
  std::memcpy(bk.prog, c->key_prog.data(), c->key_prog.size());
  for (size_t l = 0; l < c->key_leaves.size(); l++) bk.leaves[l] = leaf_desc(c->key_leaves[l]);
  return FGPU_OK;
}

// AggFuncPushDown (logicalplan/optimize.go:166-193) + MaxAgg (expr/filter.go:156-207): a global Max(column)
// directly above the scan, without filter, turns into a row-group filter that memoises the largest chunk
// maximum seen so far, in scan order, and only lets row groups through that exceed it.
struct MaxPushDown {
  const std::string* column = nullptr;  // nullptr: the plan is not a global Max(column)
  bool have = false;
  int64_t max_i = 0;
  double max_f = 0;

  // false: the row group cannot raise the maximum (L0 Arrow records are never filtered, lsm.go:420-427)
  bool admit(const VisibleRG& v) {
    if (!column || v.part->arrow) return true;
    auto it = v.rg->cols.find(*column);
    if (it == v.rg->cols.end()) return false;  // no such field in this row group: nothing to contribute
    const ChunkHost& ch = it->second;
    if (ch.null_count >= 0 && uint64_t(ch.null_count) == v.rg->n_rows) return false;
    if (!ch.has_minmax || (ch.phys != PT_INT64 && ch.phys != PT_DOUBLE)) return true;
    bool greater;
    if (ch.phys == PT_INT64) {
      greater = !have || ch.max_bits > max_i;
      if (greater) max_i = ch.max_bits;
    } else {
      double mx;
      std::memcpy(&mx, &ch.max_bits, 8);
      greater = !have || mx > max_f;
      if (greater) max_f = mx;
    }
    if (greater) have = true;
    return greater;
  }
};

// What the chunk statistics of one row group decide about one leaf (LM_EVAL: undecided).
uint8_t leaf_mode(const Compiled& c, const LeafHost& lh, const VisibleRG& v) {
  auto it = lh.slot < 0 ? v.rg->cols.end() : v.rg->cols.find(lh.column);
  // the physical plan's rule for the rows of a row group that got this far (physicalplan/binaryscalarexpr.go:47-73)
  if (it == v.rg->cols.end()) return lh.missing_mode;
  const ChunkHost& ch = it->second;
  const uint8_t st = c.slot_types[size_t(lh.slot)];
  uint8_t mode = LM_EVAL;
  if (lh.numeric && !lh.cmp_float && !lh.null_literal && st == ST_I64 && ch.has_minmax) {
    mode = chunk_leaf_mode(lh.lo_i, lh.hi_i, lh.neg, true, ch.min_bits, ch.max_bits, ch.null_count, int64_t(v.rg->n_rows));
  } else if (st == ST_DICT && lh.op == FGPU_OP_EQ && lh.lit->lit_type == FGPU_SCALAR_STRING && ch.has_minmax_str) {
    // string equality against the chunk's bounding strings (binaryscalarexpr.go:98-104; bounds may be
    // truncated by the writer, they still bound): outside them no value can be equal
    const std::string& lit = lh.lit->lit_bytes;
    if (lit < ch.min_str || lit > ch.max_str) mode = LM_NONE;
  }
  // equality with a value the chunk's bloom filter rules out: the leaf is false on every row of the row group
  // (also under a disjunction, where the row group itself stays)
  if (mode == LM_EVAL && lh.op == FGPU_OP_EQ && !lh.null_literal && !v.part->arrow && !bloom_may_contain(ch, *lh.lit)) mode = LM_NONE;
  return mode;
}

// Row-group pruning by chunk statistics.  LSM.Scan asks the filter's TrueNegativeFilter whether a row group may
// hold matching rows before it hands the row group to the plan (index/lsm.go:401-454; expr/binaryscalarexpr.go:41-190
// compares the literal with the chunk's min/max).  Same decision here, from the footer statistics, before anything
// is uploaded: an int64 range leaf whose chunk bounds miss the range selects nothing in that row group (under a
// conjunction the row group is dropped: never uploaded, never scanned); bounds inside the range of a chunk without
// NULLs select every row, and the leaf's column is then not read there.  `base`: the slots needed regardless of the
// filter.
void prune_row_groups(const QueryPlan& q, const Switches& w, const std::vector<uint8_t>& base, Compiled* c) {
  const bool conj = c->qd.n_filter_prog > 0 && c->qd.filter_kind == FK_AND;
  const bool prune_on = !w.no_prune;
  MaxPushDown max_agg;
  if (prune_on && q.kind == FGPU_PLAN_AGGREGATE && q.group_by.empty() && q.aggs.size() == 1 && q.aggs[0].func == FGPU_AGG_MAX &&
      q.filter < 0 && q.exprs[size_t(q.aggs[0].expr)].kind == FGPU_EXPR_COLUMN)
    max_agg.column = &q.exprs[size_t(q.aggs[0].expr)].name;
  std::vector<VisibleRG> kept;
  for (VisibleRG& v : c->rgs) {
    if (!max_agg.admit(v)) continue;
    // Parquet parts: the reference's own row-group filter first (L0 Arrow records are never filtered, lsm.go:420-427)
    if (prune_on && !v.part->arrow && q.filter >= 0 && !rg_may_match(q, q.filter, *v.rg)) continue;
    bool drop = false;
    for (size_t l = 0; l < c->leaves.size() && prune_on; l++) {
      v.leaf_mode[l] = leaf_mode(*c, c->leaves[l], v);
      if (conj && v.leaf_mode[l] == LM_NONE) drop = true;
    }
    if (drop) continue;
    // a boolean key's leaf decided LM_NONE makes the key false on the row group: the row group stays
    for (size_t l = 0; l < c->key_leaves.size() && prune_on; l++) v.key_leaf_mode[l] = leaf_mode(*c, c->key_leaves[l], v);
    for (size_t s = 0; s < c->slot_names.size(); s++) {
      bool needed = base[s] != 0;
      for (size_t l = 0; l < c->leaves.size() && !needed; l++)
        if (c->leaves[l].slot == int(s) && v.leaf_mode[l] == LM_EVAL) needed = true;
      for (size_t l = 0; l < c->key_leaves.size() && !needed; l++)
        if (c->key_leaves[l].slot == int(s) && v.key_leaf_mode[l] == LM_EVAL) needed = true;
      if (!needed || !c->slot_needed[s]) v.skip_slots |= 1ull << s;
    }
    kept.push_back(v);
  }
  c->pruned_row_groups = uint32_t(c->rgs.size() - kept.size());
  c->rgs.swap(kept);
  c->touched_rows = 0;
  for (const VisibleRG& v : c->rgs) c->touched_rows += v.rg->n_rows;
  // Every row group ruled out: nothing is scanned, but the plan keeps its full shape (keys, aggregates, table
  // slots): a rank whose time range misses the filter must still produce a partial table its peers can merge.
}

// Lazy residency: the columns this query projects are built and uploaded now (parts put with
// FGPU_PUT_BORROW_PINNED upload nothing until a query needs it; optimize.go:36-73 physical projection).
int32_t make_resident(fgpu_ctx* ctx, Table& table, Compiled* c) {
  PhaseClock pc;
  std::vector<std::pair<Part*, uint64_t>> reads;  // per part, in row-group order: bit s = some kept row group reads slot s
  for (const VisibleRG& v : c->rgs) {
    if (reads.empty() || reads.back().first != v.part) reads.push_back({v.part, 0});
    reads.back().second |= ~v.skip_slots;
  }
  // numeric columns first: their bytes are the bulk of the transfer, which then runs while the host
  // assembles the dictionary columns' run directories
  std::vector<std::pair<Part*, std::string>> cols;
  for (int pass = 0; pass < 2; pass++) {
    for (auto& [part, read] : reads) {
      for (size_t si = 0; si < c->slot_names.size(); si++) {
        const std::string& name = c->slot_names[si];
        if ((c->slot_types[si] == ST_DICT) != (pass == 1) || !((read >> si) & 1)) continue;
        if (std::find(part->columns.begin(), part->columns.end(), name) == part->columns.end()) continue;
        cols.push_back({part, name});
      }
    }
  }
  UploadStats st;
  const int32_t rc = upload_columns(ctx, &table, cols, &st, /*refuse_unreadable=*/true);
  c->h2d_bytes += st.h2d_bytes;
  if (rc) return rc;
  if (pc.on && c->h2d_bytes) {
    char buf[128];
    snprintf(buf, sizeof buf, " build=%.0fus enqueue=%.0fus bytes=%llu", st.build_us, st.enqueue_us, (unsigned long long)c->h2d_bytes);
    pc.line = buf;
    pc.flush("residency");
  }
  return FGPU_OK;
}

// shared-memory ring of the scan kernel: stage every numeric slot's PLAIN slice (up to kMaxStagePlain)
// and the chunk seeds of every hybrid stream (up to kMaxStageSeeds); the rest is read from HBM directly
void stage_slots(Compiled* c) {
  QueryDesc& qd = c->qd;
  for (int s = 0; s < kMaxSlots; s++) {
    qd.slot_plain_stage[s] = -1;
    qd.slot_seed_stage[s][0] = qd.slot_seed_stage[s][1] = -1;
  }
  for (int s = 0; s < qd.n_slots; s++) {
    bool any_plain = false, any_vals = false, any_def = false;
    if (!c->slot_needed[size_t(s)]) continue;
    for (const VisibleRG& v : c->rgs) {
      auto it = v.rg->cols.find(c->slot_names[size_t(s)]);
      if (it == v.rg->cols.end() || ((v.skip_slots >> s) & 1)) continue;
      const ChunkDesc& d = it->second.desc;
      if (d.kind == CK_PLAIN64 && !d.has_nulls) any_plain = true;
      if (d.kind == CK_DICT_STR || d.kind == CK_DICT64) any_vals = true;
      if (d.has_nulls) any_def = true;
    }
    if (any_plain && qd.n_stage_plain < kMaxStagePlain) {
      qd.slot_plain_stage[s] = int8_t(qd.n_stage_plain);
      qd.stage_plain_slot[qd.n_stage_plain++] = uint8_t(s);
    }
    for (int is_def = 0; is_def < 2; is_def++) {  // the values' stream, then the definition levels'
      if (!(is_def ? any_def : any_vals) || qd.n_stage_seeds >= kMaxStageSeeds) continue;
      qd.slot_seed_stage[s][is_def] = int8_t(qd.n_stage_seeds);
      qd.stage_seed_slot[qd.n_stage_seeds] = uint8_t(s);
      qd.stage_seed_is_def[qd.n_stage_seeds++] = uint8_t(is_def);
    }
  }
}

// Operand-stack depth of prog[off, off + len): the kernel evaluates aggregate and group-by expressions on a stack of
// three shared-memory vectors.
int prog_depth(const std::vector<ProgOp>& prog, size_t off, size_t len) {
  int depth = 0, maxd = 0;
  for (size_t p = off; p < off + len; p++) {
    depth += (prog[p].op == PO_LOAD || prog[p].op == PO_CONST) ? 1 : -1;
    maxd = std::max(maxd, depth);
  }
  return maxd;
}

// Whether every kept row group has every column of expression `node`; if not, *missing is the first one lacking.
bool in_every_row_group(const QueryPlan& q, int node, const std::vector<VisibleRG>& rgs, std::string* missing) {
  std::vector<std::string> cols;
  collect_columns(q, node, &cols);
  for (const VisibleRG& v : rgs)
    for (auto& n : cols)
      if (!v.rg->cols.count(n)) {
        *missing = n;
        return false;
      }
  return true;
}

// Aggregate programs, in qd.prog in aggregate order.
int32_t compile_aggregates(const QueryPlan& q, const std::map<std::string, int>& slot_of, Compiled* c, std::vector<ProgOp>* prog) {
  QueryDesc& qd = c->qd;
  if (q.aggs.size() > size_t(kMaxAggs)) return fail(FGPU_ERR_UNSUPPORTED, "too many aggregates");
  size_t cells = 0;  // stored cells and Counts: a Unique takes two (see UniqueCell)
  for (const fgpu_agg& g : q.aggs) cells += g.func == FGPU_AGG_UNIQUE ? 2 : 1;
  if (cells > size_t(kMaxAggs)) return fail(FGPU_ERR_UNSUPPORTED, "too many aggregates");
  qd.n_aggs = int32_t(cells);
  for (size_t a = 0, cell = 0; a < q.aggs.size(); a++) {
    AggDesc& ad = qd.aggs[cell];
    int f = q.aggs[a].func;
    if (f != FGPU_AGG_SUM && f != FGPU_AGG_MIN && f != FGPU_AGG_MAX && f != FGPU_AGG_COUNT && f != FGPU_AGG_UNIQUE)
      return fail(FGPU_ERR_UNSUPPORTED, std::string("aggregate function not supported on the GPU path: ") + agg_string(f));
    const bool unique = f == FGPU_AGG_UNIQUE;
    // a NULL row decides a Unique, and expressions do not track NULLs
    if (unique && q.exprs[size_t(q.aggs[a].expr)].kind != FGPU_EXPR_COLUMN)
      return fail(FGPU_ERR_UNSUPPORTED, "unique over an expression is not supported on the GPU path");
    ad.func = uint8_t(unique ? FGPU_AGG_MIN : f);
    bool any_float = false, any_int_col = false;
    size_t off = prog->size();
    int32_t rc = compile_agg_expr(q, q.aggs[a].expr, slot_of, *c, prog, &any_float, &any_int_col);
    if (rc) return rc;
    // the reference refuses Unique over float64 when it executes: the caller keeps the plan on its own operators
    if (unique && any_float) return fail(FGPU_ERR_UNSUPPORTED, "unique is defined for int64 columns only");
    if (any_float && any_int_col) return fail(FGPU_ERR_UNSUPPORTED, "arithmetic mixes int64 and float64 columns");
    if (any_float) {  // integer literals take part as doubles
      for (size_t p = off; p < prog->size(); p++)
        if ((*prog)[p].op == PO_CONST && (*prog)[p].slot == 0) {
          double d = double((*prog)[p].imm);
          std::memcpy(&(*prog)[p].imm, &d, 8);
        }
    }
    ad.is_float = any_float;
    ad.prog_off = uint8_t(off);
    ad.prog_len = uint8_t(prog->size() - off);
    // the aggregated column must exist in every record (aggregate.go:367-380)
    std::string missing;
    if (!in_every_row_group(q, q.aggs[a].expr, c->rgs, &missing))
      return fail(FGPU_ERR_NOT_FOUND, "aggregate field(s) not found [\"" + missing + "\"], aggregations are not possible without it");
    if (unique) {  // the Min cell, then the Max cell over the same program
      ad.unique = UC_LO;
      qd.aggs[cell + 1] = ad;
      qd.aggs[cell + 1].func = FGPU_AGG_MAX;
      qd.aggs[cell + 1].unique = UC_HI;
    }
    cell += unique ? 2 : 1;
  }
  // every aggregate's columns are looked up before any program is sized or its depth checked
  if (prog->size() > size_t(kMaxProg)) return fail(FGPU_ERR_UNSUPPORTED, "aggregate expressions too large");
  for (size_t p = 0; p < prog->size(); p++) qd.prog[p] = (*prog)[p];
  for (int a = 0; a < qd.n_aggs; a++)
    if (prog_depth(*prog, qd.aggs[a].prog_off, qd.aggs[a].prog_len) > 3)
      return fail(FGPU_ERR_UNSUPPORTED, "aggregate expression nests too deeply for the GPU path");
  return FGPU_OK;
}

// One result key column of the plan (slot -1: a computed or boolean key).
void add_key(Compiled* c, Table& table, const std::string& name, uint8_t type, int slot, bool is_bool = false) {
  KeyOut ko;
  ko.name = name;
  ko.is_bool = is_bool;
  ko.is_int64 = !is_bool && type != ST_DICT;
  ko.is_float = type == ST_F64;
  if (!ko.is_int64 && !is_bool) ko.dict = &table.dicts[name];  // (a column whose every row group was pruned was never built: empty dictionary)
  c->keys.push_back(std::move(ko));
  c->key_slots.push_back(slot);
}

// Filter -> Projection(columns): the resolved columns are the output of a rows plan, no table.
int32_t project_rows(const Columns& k, Table& table, Compiled* c) {
  if (k.key_names.size() > size_t(kMaxOut)) return fail(FGPU_ERR_UNSUPPORTED, "too many projected columns");
  c->qd.n_out = int32_t(k.key_names.size());
  for (size_t i = 0; i < k.key_names.size(); i++) {
    const int slot = k.slot_of.at(k.key_names[i]);
    c->qd.out_slot[i] = uint8_t(slot);
    add_key(c, table, k.key_names[i], c->slot_types[size_t(slot)], slot);
  }
  return FGPU_OK;
}

// Hash-table slots for `groups` groups: the smallest power of two >= groups, from kMinHashSlots up to kMaxHashSlots
// (beyond that a scan or a merge reports an overflow).
constexpr uint64_t kMinHashSlots = 1024, kMaxHashSlots = 1ull << 28;
uint32_t hash_slots(uint64_t groups) {
  uint64_t cap = kMinHashSlots;
  while (cap < groups && cap < kMaxHashSlots) cap <<= 1;
  return uint32_t(cap);
}

// Group keys (dictionary and int64 columns, computed int64 keys, whose programs follow the aggregates' in qd.prog, and
// boolean Distinct keys, which key like a dictionary column of two values) and the aggregate table: dense over the
// dictionary ids when every key is a dictionary or boolean key and the product of their radices is at most kDenseMax,
// a hash table of packed keys otherwise.
int32_t table_shape(const QueryPlan& q, const Columns& k, Table& table, std::vector<ProgOp>* prog, Compiled* c) {
  QueryDesc& qd = c->qd;
  qd.n_keys = int32_t(k.key_names.size());
  c->dense_radix.assign(k.key_names.size(), 0);
  bool all_dict = true;
  long double product = 1;
  for (size_t i = 0; i < k.key_names.size(); i++) {
    const std::string& name = k.key_names[i];
    const auto kx = k.key_expr.find(name);
    if (kx != k.key_expr.end()) {  // computed int64 key
      bool any_float = false, any_int_col = false;
      const size_t off = prog->size();
      int32_t rc = compile_agg_expr(q, kx->second, k.slot_of, *c, prog, &any_float, &any_int_col);
      if (rc) return rc;
      if (any_float) return fail(FGPU_ERR_UNSUPPORTED, "float64 group-by expressions are not supported");
      if (prog->size() > size_t(kMaxProg) || prog->size() - off > 255) return fail(FGPU_ERR_UNSUPPORTED, "group-by expression too large");
      if (prog_depth(*prog, off, prog->size() - off) > 3) return fail(FGPU_ERR_UNSUPPORTED, "group-by expression nests too deeply for the GPU path");
      for (size_t p = off; p < prog->size(); p++) qd.prog[p] = (*prog)[p];
      std::string missing;
      if (!in_every_row_group(q, kx->second, c->rgs, &missing)) return fail(FGPU_ERR_NOT_FOUND, "group-by expression column not found: " + missing);
      qd.keys[i].prog_off = uint8_t(off);
      qd.keys[i].prog_len = uint8_t(prog->size() - off);
    }
    if (k.bool_key.count(name)) {  // a two-entry code key (compile_bool_keys filled its program)
      add_key(c, table, name, ST_DICT, -1, /*is_bool=*/true);
      c->dense_radix[i] = 3;  // 0 NULL (never), 1 false, 2 true
      product *= 3;
      qd.keys[i].slot = 0xff;
      qd.keys[i].is_int64 = 0;
      continue;
    }
    const int slot = kx != k.key_expr.end() ? -1 : k.slot_of.at(name);
    const uint8_t type = slot < 0 ? uint8_t(ST_I64) : c->slot_types[size_t(slot)];
    if (type == ST_F64) return fail(FGPU_ERR_UNSUPPORTED, "float64 group-by columns are not supported");
    add_key(c, table, name, type, slot);
    if (type == ST_DICT) c->dense_radix[i] = c->keys.back().dict->cardinality() + 1;
    if (type != ST_DICT) all_dict = false;
    product *= type == ST_DICT ? (long double)c->dense_radix[i] : 1e18L;
    qd.keys[i].slot = uint8_t(slot < 0 ? 0xff : slot);
    qd.keys[i].is_int64 = type != ST_DICT;
  }
  long double bound = std::min<long double>(product, (long double)std::max<uint64_t>(c->total_rows, 1));
  c->group_bound = uint64_t(bound);
  const uint64_t kDenseMax = 1ull << 22;
  if (all_dict && product <= (long double)kDenseMax) {
    qd.table_mode = TM_DENSE;
    qd.key_words = 1;
    uint64_t stride = 1;
    for (size_t k = c->keys.size(); k-- > 0;) {
      qd.keys[k].dense_stride = uint32_t(stride);
      stride *= c->dense_radix[k];
    }
    qd.table_slots = uint32_t(std::max<uint64_t>(stride, 1));
    return FGPU_OK;
  }
  qd.table_mode = TM_HASH;
  int word = 0, used = 0;
  for (size_t k = 0; k < c->keys.size(); k++) {
    if (c->keys[k].is_int64) continue;
    int bits = std::max(1, bit_width_u32(c->dense_radix[k] - 1));
    if (used + bits > 64) { word++; used = 0; }
    qd.keys[k].word = uint8_t(word);
    qd.keys[k].shift = uint8_t(used);
    qd.keys[k].bits = uint32_t(bits);
    used += bits;
  }
  int words = (used > 0 || word > 0) ? word + 1 : 0;
  for (size_t k = 0; k < c->keys.size(); k++) {
    if (!c->keys[k].is_int64) continue;
    qd.keys[k].word = uint8_t(words++);
    qd.keys[k].shift = 0;
    qd.keys[k].bits = 64;
  }
  if (words > kMaxKeyWords) return fail(FGPU_ERR_UNSUPPORTED, "group key wider than the packed-key limit");
  qd.key_words = std::max(words, 1);
  qd.table_slots = hash_slots(2 * c->group_bound);
  return FGPU_OK;
}

// An aggregate that loads one column as it is (no arithmetic).
bool plain_load(const QueryDesc& qd, int a) { return qd.aggs[a].prog_len == 1 && qd.prog[qd.aggs[a].prog_off].op == PO_LOAD; }

// fused fast path of k_scan: conjunction of numeric leaves, dense dictionary keys, simple aggregates
bool fast_path_ok(const Compiled& c, const Switches& w) {
  const QueryDesc& qd = c.qd;
  if (w.no_fast || c.has_bool_keys() || c.has_unique() || qd.table_mode != TM_DENSE || (qd.n_filter_prog != 0 && qd.filter_kind != FK_AND) ||
      qd.n_leaves > 2 || qd.n_keys > 3)
    return false;
  for (int l = 0; l < qd.n_leaves; l++) {
    const LeafHost& lh = c.leaves[size_t(l)];
    if (lh.slot >= 0 && (c.slot_types[size_t(lh.slot)] == ST_DICT || lh.null_literal)) return false;
  }
  int stored = 0;
  for (int a = 0; a < qd.n_aggs; a++) {
    if (qd.aggs[a].func == FGPU_AGG_COUNT) continue;
    stored++;
    if (!plain_load(qd, a)) return false;
  }
  return stored <= 2;
}

// k_scan: vector length, ring depth and the per-warp shared-memory layout
void scan_layout(const Switches& w, Compiled* c) {
  QueryDesc& qd = c->qd;
  int vl = w.vl, ring = w.ring;
  bool any_expr = false;
  for (int k = 0; k < qd.n_keys; k++)
    if (qd.keys[k].prog_len && !qd.keys[k].is_bool) any_expr = true;
  const bool bool_keys = c->has_bool_keys();  // leafw holds the key leaves' bits once the selection is done
  for (int a = 0; a < qd.n_aggs; a++)
    if (qd.aggs[a].func != FGPU_AGG_COUNT && !plain_load(qd, a)) any_expr = true;
  auto r128 = [](size_t x) { return (x + 127) & ~size_t(127); };
  for (;;) {
    size_t off = r128(size_t(ring) * 8);
    size_t slot = r128(size_t(qd.n_stage_plain) * vl * 8 + size_t(qd.n_stage_seeds) * sizeof(Seed));
    if (slot == 0) slot = 128;
    qd.slot_bytes = uint32_t(slot);
    qd.wr_ring = uint32_t(off); off += size_t(ring) * slot;
    qd.wr_act = uint32_t(off); off = r128(off + size_t(vl / 32) * 4);
    qd.wr_leaf = uint32_t(off); off = r128(off + ((qd.n_filter_prog > 0 && qd.filter_kind != FK_AND) || bool_keys ? size_t(vl) * 4 : 0));
    qd.wr_slot = uint32_t(off); off = r128(off + size_t(vl) * 4);
    qd.wr_keyw = uint32_t(off); off = r128(off + (qd.table_mode == TM_HASH ? size_t(qd.key_words) * vl * 8 : 0));
    qd.wr_tmp1 = uint32_t(off); off = r128(off + (any_expr ? size_t(vl) * 8 : 0));
    qd.wr_tmp2 = uint32_t(off); off = r128(off + (any_expr ? size_t(vl) * 16 : 0));
    qd.wr_acc = uint32_t(off); off = r128(off + size_t(qd.n_aggs) * 32 * 8 + 16 + 32 * 4 + 32 * 4 + (qd.table_mode == TM_HASH ? size_t(qd.key_words) * 32 * 8 : 0));
    qd.wr_cdesc = uint32_t(off); off = r128(off + size_t(std::max(qd.n_slots, 1)) * sizeof(ChunkDesc));
    qd.wr_clrt = uint32_t(off); off = r128(off + size_t(std::max(qd.n_leaves, 1)) * sizeof(LeafRt));
    qd.wr_fplan = uint32_t(off); off = r128(off + 512);
    qd.wr_iplan = uint32_t(off); off = r128(off + 8 + 16 * size_t(kMaxStagePlain + kMaxStageSeeds));
    c->bool_keys.wr_keys = uint32_t(off); off = r128(off + (bool_keys ? sizeof(BoolKeys) + c->key_leaves.size() * sizeof(LeafRt) : 0));
    qd.wr_bytes = uint32_t(off);
    if (size_t(qd.wr_bytes) * (kVecThreads / 32) <= 200 * 1024 || vl == 128) break;
    vl /= 2;  // many staged columns / wide keys: shorter vectors
  }
  qd.vl = vl;
  qd.n_ring = ring;
  qd.fast_ok = fast_path_ok(*c, w) ? 1 : 0;
}

// Resolves the plan against the visible row groups and fills everything of QueryDesc that does
// not need device memory.  The phases run in this order, and so do their refusals.
int32_t compile(fgpu_ctx* ctx, const QueryPlan& q, uint64_t tx, const Switches& w, Compiled* c) {
  Table& table = ctx->tables[q.table];  // a table without parts scans nothing (empty LSM)
  for (auto& p : table.parts) {
    if (p->tx > tx) continue;  // index/lsm.go:416
    for (auto& rg : p->rgs) {
      c->rgs.push_back({p.get(), &rg});
      c->total_rows += rg.n_rows;
    }
  }
  QueryDesc& qd = c->qd;
  qd.tile_rows = ctx->tile_rows;
  if (c->rgs.empty()) {  // nothing to scan: no records, exactly like an Iterator over an empty LSM
    qd.table_mode = TM_DENSE;
    qd.key_words = 1;
    qd.table_slots = 1;
    return FGPU_OK;
  }
  Columns k;
  int32_t rc = resolve_columns(q, table, c, &k);
  if (rc) return rc;
  rc = compile_predicate(q, w, k.slot_of, c);
  if (rc) return rc;
  rc = compile_bool_keys(q, k, c);
  if (rc) return rc;
  prune_row_groups(q, w, q.kind == FGPU_PLAN_FILTER ? std::vector<uint8_t>(c->slot_names.size(), 1) : k.value_slots(q, false), c);
  rc = make_resident(ctx, table, c);
  if (rc) return rc;
  stage_slots(c);
  std::vector<ProgOp> prog;
  rc = compile_aggregates(q, k.slot_of, c, &prog);
  if (rc) return rc;
  qd.n_rg = int32_t(c->rgs.size());
  if (q.kind == FGPU_PLAN_FILTER) return project_rows(k, table, c);
  rc = table_shape(q, k, table, &prog, c);
  if (rc) return rc;
  scan_layout(w, c);
  return FGPU_OK;
}

size_t table_layout(const QueryDesc& qd, size_t* off_aggs, size_t* off_tags, size_t* off_keys) {
  size_t S = qd.table_slots;
  int n_stored = 0;
  for (int a = 0; a < qd.n_aggs; a++)
    if (qd.aggs[a].func != FGPU_AGG_COUNT) n_stored++;
  *off_aggs = S * 8;
  *off_tags = S * 8 * size_t(1 + n_stored);
  size_t tags = (qd.table_mode == TM_HASH) ? ((S * 4 + 7) & ~size_t(7)) : 0;
  *off_keys = *off_tags + tags;
  size_t keys = (qd.table_mode == TM_HASH) ? S * 8 * size_t(qd.key_words) : 0;
  return *off_keys + keys;
}

void bind_table(QueryDesc* qd, uint8_t* base) {
  size_t off_aggs, off_tags, off_keys;
  table_layout(*qd, &off_aggs, &off_tags, &off_keys);
  size_t S = qd->table_slots;
  qd->t_rows = reinterpret_cast<unsigned long long*>(base);
  int pos = 0;
  for (int a = 0; a < kMaxAggs; a++) qd->t_agg[a] = nullptr;
  for (int a = 0; a < qd->n_aggs; a++) {
    if (qd->aggs[a].func == FGPU_AGG_COUNT) continue;
    qd->t_agg[a] = reinterpret_cast<long long*>(base + off_aggs + size_t(pos) * S * 8);
    pos++;
  }
  qd->t_tag = qd->table_mode == TM_HASH ? reinterpret_cast<uint32_t*>(base + off_tags) : nullptr;
  qd->t_keys = qd->table_mode == TM_HASH ? reinterpret_cast<unsigned long long*>(base + off_keys) : nullptr;
}

void bind_finalize(FinalizeDesc* fd, const QueryDesc& qd) {  // the table bind_table placed
  fd->t_rows = qd.t_rows;
  for (int a = 0; a < kMaxAggs; a++) fd->t_agg[a] = qd.t_agg[a];
  fd->t_tag = qd.t_tag;
  fd->t_keys = qd.t_keys;
}

int32_t finalize_dense_host(fgpu_result* res, ExecCache& x);

// FROSTGPU_COMM_TIMEOUT_MS: how long a collective Execute waits for its peers (default 10 s).  It changes no plan, so
// it is not one of the Switches.
uint64_t comm_timeout_ns() {
  const char* to = getenv("FROSTGPU_COMM_TIMEOUT_MS");
  return uint64_t(to ? std::max(1, atoi(to)) : 10000) * 1000000ull;
}

// First half of the exchange, enqueued behind the scan: this rank's partial table goes into slot [rank] of every
// rank's mailbox, then the flags are raised (comm.cu).
int32_t comm_push(fgpu_ctx* ctx, const void* table, size_t table_bytes, uint64_t* out_seq, uint64_t* out_bytes) {
  Comm& cm = ctx->comm;
  if (!cm.open) return fail(FGPU_ERR_INVALID, "collective Execute without an open communicator (fgpu_comm_open)");
  const size_t bytes = (table_bytes + 15) & ~size_t(15);
  if (bytes > cm.slot_bytes) return fail(FGPU_ERR_UNSUPPORTED, "partial table (" + std::to_string(bytes) + " bytes) larger than the exchange slot");
  const uint64_t seq = ++cm.seq, set = seq & 1u;
  CommPush p{};
  p.done = reinterpret_cast<unsigned int*>(cm.mailbox + 2048);  // (inside the zeroed header region, behind the flags)
  p.src = static_cast<const uint8_t*>(table);
  p.bytes = bytes;
  p.seq = seq;
  p.n = cm.n;
  for (int r = 0; r < cm.n; r++) {
    p.dst[r] = cm.peer[r] + cm.data_off(set, cm.rank);
    p.flag[r] = reinterpret_cast<unsigned long long*>(cm.peer[r] + cm.flag_off(set, cm.rank));
  }
  CUDA_TRY(launch_comm_push(p, ctx->sm_count, ctx->stream));
  *out_seq = seq;
  *out_bytes = bytes;
  return FGPU_OK;
}

// Second half: wait for every rank's flag; dense tables are then folded from the n mailbox slots into `table`
// itself (it holds the FINAL table afterwards).  Hash tables: the caller merges the slots with k_merge.
int32_t comm_wait_merge(fgpu_ctx* ctx, const QueryDesc& qd, void* table, uint64_t seq, uint64_t bytes) {
  Comm& cm = ctx->comm;
  const uint64_t set = seq & 1u;
  CommWait w{};
  w.flags = reinterpret_cast<const unsigned long long*>(cm.mailbox + cm.flag_off(set, 0));
  w.seq = seq;
  w.bytes = qd.table_mode == TM_DENSE ? bytes : 0;  // hash tables: sized per rank, checked by hash_partial_slots
  w.timeout_ns = comm_timeout_ns();
  w.counters = qd.counters;
  w.n = cm.n;
  CUDA_TRY(launch_comm_wait(w, ctx->stream));
  if (qd.table_mode == TM_DENSE) {
    CommMerge m{};
    m.n = cm.n;
    for (int r = 0; r < cm.n; r++) m.src[r] = cm.mailbox + cm.data_off(set, r);
    QueryDesc q2 = qd;
    bind_table(&q2, static_cast<uint8_t*>(table));
    CUDA_TRY(launch_merge_dense(q2, m, ctx->stream));
  }
  return FGPU_OK;
}

int32_t comm_check(unsigned long long code) {
  if (code == 1) return fail(FGPU_ERR_CUDA, "collective Execute: a peer did not deliver its partial table within the timeout");
  if (code == 2) return fail(FGPU_ERR_UNSUPPORTED, "collective Execute: partial table shapes differ between ranks (dictionaries not preloaded identically?)");
  return FGPU_OK;
}

// Hash mode: a rank sizes its partial table from its own visible rows, so the ranks' tables differ in size.  Behind
// the wait, each rank's pushed byte count is read from the flags of this set (one copy, one synchronisation); it must
// be this plan's table_layout at a power-of-two slot count, whose slot count goes to src_slots[r].
int32_t hash_partial_slots(fgpu_ctx* ctx, const QueryDesc& qd, uint64_t seq, uint32_t* src_slots) {
  Comm& cm = ctx->comm;
  CUDA_TRY(ctx->ensure_scratch(size_t(kMaxRanks) * 16));
  unsigned long long* flags = reinterpret_cast<unsigned long long*>(ctx->scratch);
  CUDA_TRY(cudaMemcpyAsync(flags, cm.mailbox + cm.flag_off(seq & 1u, 0), size_t(cm.n) * 16, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  for (int r = 0; r < cm.n; r++) {
    if (flags[2 * r] < seq) return comm_check(1);  // k_comm_wait gave up on this peer
    src_slots[r] = 0;
    for (uint64_t S = kMinHashSlots; S <= kMaxHashSlots && !src_slots[r]; S <<= 1) {
      QueryDesc q = qd;
      q.table_slots = uint32_t(S);
      size_t off_aggs, off_tags, off_keys;
      if (((table_layout(q, &off_aggs, &off_tags, &off_keys) + 15) & ~size_t(15)) == flags[2 * r + 1]) src_slots[r] = uint32_t(S);
    }
    if (!src_slots[r]) return comm_check(2);
  }
  return FGPU_OK;
}

// k_finalize with max_out == 0 only counts the groups of the table, into *out.
cudaError_t launch_count_groups(FinalizeDesc fd, unsigned int* out, cudaStream_t s) {
  fd.out_count = out;
  fd.max_out = 0;
  fd.out_keys = nullptr;
  fd.out_aggs = nullptr;
  fd.out_rows = nullptr;
  return launch_finalize(fd, s);
}

// Tail of a cached Execute: compact the (final) dense table into result columns on the device and bring them back.
// The result image is written by the kernel straight into a page-locked block of the context's pool (host memory the
// device addresses directly): no copy operation, and the block later travels to the Arrow consumer as it is.
int32_t cached_tail(fgpu_ctx* ctx, ExecCache& x) {
  cudaStream_t s = ctx->stream;
  if (!x.pinned) {
    x.pinned = PinnedBlock(ctx->pinned, x.out_bytes);
    if (!x.pinned) return fail(FGPU_ERR_OOM, "page-locked memory for the result image");
  }
  // k_finalize_dense writes the block over PCIe itself: 22 us of kernel time for 400 KB against 4 + 9 for kernel + copy
  // engine, but the Execute is 8 us shorter end to end without the copy operation behind the kernel (measured)
  x.dout.out = x.pinned.get();
  CUDA_TRY(launch_finalize_dense(x.dout, s));
  return FGPU_OK;
}

// Collective tail of a cached Execute (cached plans have dense tables): ONE launch waits for the peers' flags, folds
// the n partial tables of this rank's mailbox and compacts the result into the page-locked block (synchronize.go:16-53
// + the final aggregate of physicalplan.go:438-471).
int32_t cached_merge_tail(fgpu_ctx* ctx, ExecCache& x, uint64_t seq, uint64_t bytes) {
  Comm& cm = ctx->comm;
  const uint64_t set = seq & 1u;
  DenseOut& f = x.dout;
  f.n_src = cm.n;
  for (int r = 0; r < cm.n; r++) f.src[r] = cm.mailbox + cm.data_off(set, r);
  f.flags = reinterpret_cast<const unsigned long long*>(cm.mailbox + cm.flag_off(set, 0));
  f.seq = seq;
  f.bytes = bytes;
  f.timeout_ns = comm_timeout_ns();
  f.err = x.qd.counters + 3;
  const int32_t rc = cached_tail(ctx, x);
  f.n_src = 0;
  return rc;
}

// k_runs_prefix or k_table_init, the other aggregate-scan launches, k_scan; ev[1] and ev[2] bracket the scan kernels
// (with k_runs_prefix among them).
int32_t launch_aggregate_scan(fgpu_ctx* ctx, const QueryDesc& qd, const QueryDesc* qdesc_dev, const ScanLaunch& L) {
  cudaStream_t s = ctx->stream;
  if (!L.prefix) CUDA_TRY(launch_table_init(qd, s));
  CUDA_TRY(cudaEventRecord(ctx->ev[1], s));
  if (L.prefix) CUDA_TRY(launch_runs_prefix(L.pd, ctx->sm_count, s));
  if (L.runs) CUDA_TRY(launch_runs_tma(L.rd, L.runs_nl, L.runs_nk, L.runs_na, ctx->sm_count, s));
  if (L.tile) CUDA_TRY(launch_tile_agg(L.td, ctx->sm_count, s));
  CUDA_TRY(launch_scan(qdesc_dev, qd, ctx->sm_count, s));
  CUDA_TRY(cudaEventRecord(ctx->ev[2], s));
  return FGPU_OK;
}

// End of an Execute's scan launches: one synchronisation, the staging of this Execute's uploads released behind it,
// then the scan kernels' time (ev[1] to ev[2]) and, with `total`, the device time of the whole Execute (ev[0] to ev[3],
// which is recorded here behind the last launch).
int32_t finish_scan(fgpu_ctx* ctx, PhaseClock& pc, fgpu_stats& st, bool total) {
  if (total) CUDA_TRY(cudaEventRecord(ctx->ev[3], ctx->stream));
  pc.mark("launch");
  CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  pc.mark("sync");
  release_staging(ctx);
  float ms = 0;
  CUDA_TRY(cudaEventElapsedTime(&ms, ctx->ev[1], ctx->ev[2]));
  st.scan_kernel_ms = ms;
  if (total) {
    CUDA_TRY(cudaEventElapsedTime(&ms, ctx->ev[0], ctx->ev[3]));
    st.total_device_ms = ms;
  }
  return FGPU_OK;
}

// Re-issues the launches of a cached plan (see ExecCache): table init, scans, one copy back, one synchronisation.
// collective: 0 no exchange, 1 push + wait + merge in one go, 2 push only (fgpu_query_execute_collective_begin)
int32_t run_cached(fgpu_ctx* ctx, ExecCache& x, fgpu_result* res, int collective) {
  PhaseClock pc;
  struct Tail { PhaseClock& pc; ~Tail() { pc.flush("cached"); } } tail{pc};
  cudaStream_t s = ctx->stream;
  res->stats = x.stats;
  fgpu_stats& st = res->stats;
  CUDA_TRY(cudaEventRecord(ctx->ev[0], s));
  if (int32_t rc = launch_aggregate_scan(ctx, x.qd, x.qdesc_dev, x.launch)) return rc;
  if (collective) {
    uint64_t seq = 0, bytes = 0;
    if (int32_t rc = comm_push(ctx, x.table.p, x.table_bytes, &seq, &bytes)) return rc;
    st.kernel_launches++;  // k_comm_push
    if (collective == 2) {  // the merge half follows in fgpu_query_execute_collective_end
      res->pending = true;
      res->pending_cached = &x;
      res->pending_seq = seq;
      res->pending_bytes = bytes;
      return FGPU_OK;
    }
    if (int32_t rc = cached_merge_tail(ctx, x, seq, bytes)) return rc;
  } else if (int32_t rc = cached_tail(ctx, x)) {
    return rc;
  }
  if (int32_t rc = finish_scan(ctx, pc, st, /*total=*/true)) return rc;
  const unsigned long long* counters = reinterpret_cast<const unsigned long long*>(x.pinned.get() + 32);
  st.rows_selected = counters[0];
  st.d2h_bytes += x.out_bytes;
  if (int32_t rc = comm_check(counters[3])) return rc;
  const int32_t rc = finalize_dense_host(res, x);
  pc.mark("export");
  return rc;
}

// ---- Execute planning -----------------------------------------------------------------------------------------------
// Every row group gets a row of the general tables that k_scan / k_rows read.  The specialised kernels may then take it,
// in run_scan's order; each has a planner of three steps: a query-level check that fills its plan (or says no), an
// admit step over the row group's rows of the general tables, and a layout step once every row group is placed.  Each
// plan (the general tables included) then places its tables in the Execute's descriptor block (place), binds their
// device addresses into its descriptor once the block is allocated (bind, before the block's image is copied), and says
// how many launches it issues (launches).

// The host image of an Execute's descriptor block: pieces at 16-byte aligned offsets, in the order they are added,
// copied into page-locked scratch and uploaded with one copy.  A piece without a source is left zero.
struct HostImage {
  struct Piece { const void* src; size_t bytes, off; };
  std::vector<Piece> pieces;
  size_t end = 0;
  static size_t align16(size_t x) { return (x + 15) & ~size_t(15); }
  size_t add(const void* src, size_t bytes) {
    const size_t off = align16(end);
    pieces.push_back({src, bytes, off});
    end = off + bytes;
    return off;
  }
  template <class T> size_t add(const std::vector<T>& v) { return add(v.data(), v.size() * sizeof(T)); }
  void copy_to(uint8_t* dst) const {
    for (const Piece& p : pieces)
      if (p.src && p.bytes) std::memcpy(dst + p.off, p.src, p.bytes);
  }
};

template <class T> T* dev_at(uint8_t* block, size_t off) { return reinterpret_cast<T*>(block + off); }

// The per-row-group descriptors of the specialised kernels refer to the LUT block before it has a device address: their
// pred_lut entries hold its byte offset + 1 (null: no LUT) until lut_rebase turns them into pointers.
const uint8_t* lut_ref(size_t off) { return reinterpret_cast<const uint8_t*>(uintptr_t(off) + 1); }
template <class Rg> void lut_rebase(std::vector<Rg>& rgs, const uint8_t* lut) {
  for (Rg& r : rgs)
    for (const uint8_t*& p : r.pred_lut)
      if (p) p = lut + (size_t(uintptr_t(p)) - 1);
}

// The table a specialised kernel adds to (the one k_scan adds to): its aggregate i is the query's agg_index[i].
template <class D> void bind_target(D& d, const QueryDesc& qd, const int* agg_index, int na) {
  d.t_rows = qd.t_rows;
  for (int a = 0; a < na; a++) d.t_agg[a] = qd.t_agg[agg_index[a]];
  d.counters = qd.counters;
}

struct GeneralTables {
  std::vector<ChunkDesc> chunks;  // [row group][slot]
  std::vector<LeafRt> lrt;        // [row group][leaf]
  std::vector<LeafRt> key_lrt;    // [row group][boolean key leaf]
  std::vector<uint32_t> first_tile, rg_rows;
  std::vector<uint8_t> lutbytes;                   // dictionary leaves: one result byte per global dictionary id
  std::vector<std::pair<size_t, size_t>> lut_fix;  // (index into lrt, offset into lutbytes)
  std::vector<std::pair<size_t, size_t>> key_lut_fix;  // (index into key_lrt, offset into lutbytes)
  uint32_t tiles = 0;
  int n = 0;  // row groups that stay with the general kernel
  BoolKeys bk{};
  bool has_bk = false;
  size_t o_chunks = 0, o_lrt = 0, o_first = 0, o_rows = 0, o_lut = 0, o_klrt = 0, o_bk = 0;
  GeneralTables(int n_rg, int n_slots, int n_leaves, int n_key_leaves)
      : chunks(size_t(n_rg) * std::max(n_slots, 1)), lrt(size_t(n_rg) * std::max(n_leaves, 1)), key_lrt(size_t(n_rg) * n_key_leaves),
        first_tile(size_t(n_rg) + 1), rg_rows(std::max(n_rg, 1)) {}
  void place(HostImage& img, const Compiled& c) {
    o_chunks = img.add(chunks);
    o_lrt = img.add(lrt);
    o_first = img.add(first_tile);
    o_rows = img.add(rg_rows);
    o_lut = img.add(lutbytes);
    o_klrt = img.add(key_lrt);
    has_bk = c.has_bool_keys();
    bk = c.bool_keys;
    if (has_bk) o_bk = img.add(&bk, sizeof bk);
  }
  // Returns the device address of the LUT block, which the other plans' bind steps rebase onto.
  const uint8_t* bind(uint8_t* block, QueryDesc& qd) {
    const uint8_t* lut = block + o_lut;
    for (auto& fx : lut_fix) lrt[fx.first].lut = lut + fx.second;
    for (auto& fx : key_lut_fix) key_lrt[fx.first].lut = lut + fx.second;
    if (has_bk) {
      bk.leaf_rt = dev_at<const LeafRt>(block, o_klrt);
      qd.bool_keys = dev_at<const BoolKeys>(block, o_bk);
    }
    qd.chunks = dev_at<const ChunkDesc>(block, o_chunks);
    qd.leaf_rt = dev_at<const LeafRt>(block, o_lrt);
    qd.rg_first_tile = dev_at<const uint32_t>(block, o_first);
    qd.rg_rows = dev_at<const uint32_t>(block, o_rows);
    return lut;
  }
  uint32_t launches() const { return tiles ? 1 : 0; }  // k_scan, or k_rows
};

// Fills row G.n of the general tables from row group g0 of the plan.
int32_t describe_row_group(fgpu_ctx* ctx, const QueryPlan& q, Compiled& c, int g0, GeneralTables& G, fgpu_stats& st) {
  const int n_slots = c.qd.n_slots, n_leaves = c.qd.n_leaves;
  const VisibleRG& v = c.rgs[size_t(g0)];
  const size_t g = size_t(G.n);
  for (int s = 0; s < n_slots; s++) {
    ChunkDesc d{};
    d.kind = CK_ABSENT;
    d.n_rows = v.rg->n_rows;
    auto it = ((v.skip_slots >> s) & 1) ? v.rg->cols.end() : v.rg->cols.find(c.slot_names[size_t(s)]);
    if (it != v.rg->cols.end()) {
      ChunkHost& ch = it->second;
      if (!ch.error.empty())
        return fail(FGPU_ERR_UNSUPPORTED, "column " + c.slot_names[size_t(s)] + ": " + ch.error);
      d = ch.desc;
      st.algorithmic_bytes += ch.stored_bytes;
      st.metadata_bytes += ch.meta_bytes;
    }
    G.chunks[g * n_slots + s] = d;
  }
  // the LeafRt of one leaf, stored at (*lrt)[at]; `decided`: what the statistics decided (LM_EVAL: nothing)
  auto describe_leaf = [&](LeafHost& lh, uint8_t decided, std::vector<LeafRt>* lrt, std::vector<std::pair<size_t, size_t>>* lut_fix, size_t at) {
    LeafRt rt{};
    auto it = lh.slot < 0 ? v.rg->cols.end() : v.rg->cols.find(lh.column);
    if (it == v.rg->cols.end()) {
      rt.mode = lh.missing_mode;
    } else if (c.slot_types[size_t(lh.slot)] == ST_DICT) {
      rt.mode = LM_EVAL;
      rt.null_result = (lh.op == FGPU_OP_EQ && lh.lit->lit_type == FGPU_SCALAR_NULL) ? 1 : 0;
      if (lh.lut_off == size_t(-1)) {
        // one result byte per GLOBAL dictionary id, evaluated once per distinct dictionary entry
        const GlobalDict& gd = ctx->tables[q.table].dicts[lh.column];
        lh.lut_off = G.lutbytes.size();
        G.lutbytes.resize(lh.lut_off + gd.values.size() + 1);
        for (size_t i = 0; i < gd.values.size(); i++) G.lutbytes[lh.lut_off + i] = dict_leaf_value(lh, gd.values[i]) ? 1 : 0;
      }
      lut_fix->emplace_back(at, lh.lut_off);
    } else {
      rt.mode = lh.null_literal ? LM_NONE : LM_EVAL;
    }
    if (decided != LM_EVAL) rt.mode = decided;
    (*lrt)[at] = rt;
  };
  for (int l = 0; l < n_leaves; l++) describe_leaf(c.leaves[size_t(l)], v.leaf_mode[l], &G.lrt, &G.lut_fix, g * n_leaves + l);
  const size_t nk = c.key_leaves.size();
  for (size_t l = 0; l < nk; l++) describe_leaf(c.key_leaves[l], v.key_leaf_mode[l], &G.key_lrt, &G.key_lut_fix, g * nk + l);
  return FGPU_OK;
}

// Index of `slot` in slots[0, *n), appended when missing (-1: the list is full at cap).
int find_or_add(int* slots, uint32_t* n, int cap, int slot) {
  for (uint32_t i = 0; i < *n; i++)
    if (slots[i] == slot) return int(i);
  if (*n >= uint32_t(cap)) return -1;
  slots[*n] = slot;
  return int((*n)++);
}

// A dictionary column whose runs are long enough that a 32-row step rarely holds two run ends (row_runs: the
// directory in row space; it exists when the column chunk is run-length only, NULLs included).  Short runs — a leaf
// on a column far down the sort order — are the tile-aggregate kernel's business: its per-row result byte costs one
// shared load where a cursor would move every few rows.
bool long_runs(const ChunkDesc& d, uint32_t n_rows) {
  return d.kind == CK_DICT_STR && d.row_runs != nullptr && uint64_t(d.n_row_runs) * 32 <= uint64_t(n_rows) + 1024;
}

// ---- sorted-run scan (runs_tma.cu) ----
// One launch over the qualifying row groups; a row group whose statistics already decided every leaf is flagged
// all_pass (its leaf columns are neither uploaded nor staged).
struct RunsRgCols {  // the chunks behind RunsRg::col (null: not staged)
  Part* part = nullptr;
  ChunkHost* ch[kRunsCols] = {nullptr};
};
struct RunsCand {  // a row group the sorted-run kernel admitted
  RunsRg rr{};
  RunsRgCols cols{};
};
struct RunsPlan {
  RunsDesc rd{};
  int nl = 0, nk = 0, na = 0, np = 0;
  int leaf_index[kRunsLeaves] = {0}, pred_leaf[kRunsPreds] = {0};  // query leaf behind every range / dictionary leaf
  int agg_slot[kRunsAggs] = {0}, agg_index[kRunsAggs] = {0};
  int col_slot[kRunsCols] = {0};  // slot of every distinct staged column
  std::vector<RunsRg> rgs;
  std::vector<RunsRgCols> cols;
  std::vector<uint32_t> first_span;
  size_t o_rgs = 0, o_span = 0;
  void place(HostImage& img) {
    o_rgs = img.add(rgs);
    o_span = img.add(first_span);
  }
  void bind(uint8_t* block, const uint8_t* lut, const QueryDesc& qd, ScanLaunch& L) {
    lut_rebase(rgs, lut);
    L.runs = !rgs.empty();
    L.rd = rd;
    L.rd.rgs = dev_at<const RunsRg>(block, o_rgs);
    L.rd.rg_first_span = dev_at<const uint32_t>(block, o_span);
    bind_target(L.rd, qd, agg_index, na);
    L.runs_nl = nl;
    L.runs_nk = nk;
    L.runs_na = na;
  }
  uint32_t launches() const { return rgs.empty() ? 0 : 1; }  // k_runs_tma
};

// Dense keys (up to kRunsKeys), a conjunction of int64 range leaves and of dictionary leaves (evaluated once per run),
// up to kRunsAggs Sum / Min / Max of plain columns.
bool runs_query(const Compiled& c, const QueryDesc& qd, const Switches& w, RunsPlan* P) {
  if (w.no_fast || w.no_runs || c.has_bool_keys() || c.has_unique() || qd.table_mode != TM_DENSE || (qd.n_filter_prog != 0 && qd.filter_kind != FK_AND) ||
      qd.n_keys > kRunsKeys || qd.n_leaves > kRunsLeaves + kRunsPreds)
    return false;
  RunsDesc& rd = P->rd;
  auto col_of = [&](int slot) { return uint32_t(find_or_add(P->col_slot, &rd.n_cols, kRunsCols, slot)); };
  for (int l = 0; l < qd.n_leaves; l++) {
    const LeafHost& lh = c.leaves[size_t(l)];
    const LeafDesc& ld = qd.leaves[l];
    if (lh.slot >= 0 && lh.numeric && lh.null_literal) return false;
    if (ld.slot == 0xff || qd.slot_type[ld.slot] == ST_DICT) {  // dictionary leaf, or a column absent from every row group
      if (P->np >= kRunsPreds) return false;
      P->pred_leaf[P->np++] = l;
    } else if (ld.cmp_float || ld.neg || qd.slot_type[ld.slot] != ST_I64 || P->nl >= kRunsLeaves) {
      return false;
    } else {
      P->leaf_index[P->nl] = l;
      rd.leaf_col[P->nl++] = col_of(ld.slot);
    }
  }
  for (int a = 0; a < qd.n_aggs; a++) {
    const AggDesc& ad = qd.aggs[a];
    if (ad.func == FGPU_AGG_COUNT) continue;
    if (!(ad.prog_len == 1 && qd.prog[ad.prog_off].op == PO_LOAD)) return false;
    if ((ad.func != FGPU_AGG_SUM && ad.func != FGPU_AGG_MIN && ad.func != FGPU_AGG_MAX) || P->na >= kRunsAggs) return false;
    P->agg_slot[P->na] = qd.prog[ad.prog_off].slot;
    rd.agg_col[P->na] = col_of(P->agg_slot[P->na]);
    rd.agg_func[P->na] = uint32_t(ad.func) | (ad.is_float ? 0x100u : 0u);
    P->agg_index[P->na++] = a;
  }
  P->nk = qd.n_keys;
  for (int k = 0; k < P->nk; k++) rd.stride[k] = qd.keys[k].dense_stride;
  rd.n_pred = uint32_t(P->np);
  return true;
}

bool runs_admit(RunsPlan& P, const Compiled& c, const QueryDesc& qd, const VisibleRG& v, const ChunkDesc* chunks, const LeafRt* lrt, RunsCand* out) {
  const uint32_t n_rows = v.rg->n_rows;
  if (n_rows == 0) return false;
  bool all_pass = P.nl > 0;
  for (int l = 0; l < P.nl; l++) {
    const uint8_t m = lrt[P.leaf_index[l]].mode;
    if (m != LM_ALL) all_pass = false;
    if (m == LM_NONE) return false;  // (only with pruning switched off)
  }
  RunsRg& rr = out->rr;
  rr.n_rows = n_rows;
  for (int l = 0; l < P.nl; l++) {
    const int ql = P.leaf_index[l];
    const bool all = lrt[ql].mode == LM_ALL;
    rr.lo[l] = all ? std::numeric_limits<int64_t>::min() : qd.leaves[ql].lo_i;
    rr.hi[l] = all ? std::numeric_limits<int64_t>::max() : qd.leaves[ql].hi_i;
  }
  for (int i = 0; i < P.np; i++) {  // dictionary leaves: one result per run
    const int ql = P.pred_leaf[i];
    const LeafRt& rt = lrt[ql];
    rr.pred_runs[i] = nullptr;
    if (rt.mode == LM_ALL) continue;         // decided: passes everywhere in this row group
    if (rt.mode == LM_NONE) return false;    // (only with pruning switched off)
    const ChunkDesc& d = chunks[qd.leaves[ql].slot];
    if (!long_runs(d, n_rows)) return false;
    rr.pred_runs[i] = d.row_runs;
    rr.pred_seeds[i] = d.row_seeds;
    rr.pred_n_runs[i] = d.n_row_runs;
    rr.pred_lut[i] = lut_ref(c.leaves[size_t(ql)].lut_off);
    P.rd.pred_null[i] = rt.null_result;
  }
  rr.all_pass = all_pass ? 1 : 0;
  bool any_col = false;
  out->cols.part = v.part;
  for (uint32_t i = 0; i < P.rd.n_cols; i++) {
    const ChunkDesc& d = chunks[P.col_slot[i]];
    rr.col[i] = nullptr;
    if ((v.skip_slots >> P.col_slot[i]) & 1) continue;  // a decided leaf's own column
    if (d.kind != CK_PLAIN64 || d.has_nulls) return false;
    rr.col[i] = d.values;
    out->cols.ch[i] = &v.rg->cols.at(c.slot_names[size_t(P.col_slot[i])]);
    any_col = true;
  }
  // all_pass: the leaf columns stay null (not staged).  Otherwise a decided leaf still runs its (widened) range test:
  // a staged column stands in for the one that was not uploaded (see the tile plan).
  if (!all_pass && !any_col && P.rd.n_cols > 0) return false;
  if (all_pass)  // aggregate inputs must be there
    for (int a = 0; a < P.na; a++)
      if (!rr.col[P.rd.agg_col[a]]) return false;
  for (int k = 0; k < P.nk; k++) {  // keys: run-length only, long runs
    const ChunkDesc& d = chunks[qd.keys[k].slot];
    if (!long_runs(d, n_rows)) return false;
    rr.runs[k] = d.row_runs;
    rr.seeds[k] = d.row_seeds;
    rr.n_runs[k] = d.n_row_runs;
  }
  return true;
}

// ---- prefix sums (runs_prefix.cu) ----
// Row groups of the sorted-run shape whose filter the statistics decided, without undecided dictionary leaves and with
// Sum(int64) as the only stored aggregates, are answered from prefix sums instead when their runs average at least
// kPrefixRunRows rows: then a step per group run is cheaper than reading its rows.
constexpr uint64_t kPrefixRunRows = 64;
struct PrefixPlan {
  PrefixBuildDesc bd{};
  std::vector<PrefixRg> rgs;
  std::vector<std::array<ChunkHost*, kRunsAggs>> sums;  // per row group: the chunk of every Sum input
  std::vector<Part*> parts;
  std::vector<PrefixWin> wins;
  uint64_t seg_bound = 0;  // segments at most: every run start of every key column and every window start
  uint64_t all_rows = 0;   // rows of the admitted row groups (they all pass)
  uint32_t n_sums = 1;     // distinct Sum inputs of the first row group (as the accounting counts them)
  size_t o_rgs = 0, o_wins = 0;
  void place(HostImage& img) {
    o_rgs = img.add(rgs);
    o_wins = img.add(wins);
  }
  void bind(uint8_t* block, ScanLaunch& L) {  // (k_runs_prefix's own descriptor is filled by prefix_build)
    L.prefix = !rgs.empty();
    bd.rgs = dev_at<const PrefixRg>(block, o_rgs);
    bd.wins = dev_at<const PrefixWin>(block, o_wins);
  }
  uint32_t launches() const { return rgs.empty() ? 0 : 1; }  // k_runs_prefix (the segment-table build: PrefixBuilt)
};

// After the build step: its launches, and the bytes an Execute reads per segment (entry + P[b], P[e] of every distinct
// Sum input), counted once the build's segment count is back on the host.
struct PrefixBuilt {
  const uint32_t* count = nullptr;  // page-locked: seg_off[table_slots]
  uint64_t per_seg = 0;
  uint32_t launches = 0;
  void account(fgpu_stats& st) const {
    if (count) st.algorithmic_bytes += uint64_t(*count) * per_seg;
  }
};

bool prefix_query(const Compiled& c, const RunsPlan& R, const Switches& w) {
  if (w.no_prefix || c.has_bool_keys() || c.has_unique()) return false;
  for (int a = 0; a < R.na; a++)
    if (R.rd.agg_func[a] != uint32_t(FGPU_AGG_SUM)) return false;  // Min / Max / float64 Sum stay with k_runs_tma
  return true;
}

// A row group the sorted-run kernel admitted.
bool prefix_admit(PrefixPlan& P, const RunsPlan& R, const RunsCand& rc, fgpu_stats& st) {
  const RunsRg& rr = rc.rr;
  if (R.nl > 0 && !rr.all_pass) return false;  // (the kernel treats a launch without range leaves as all-pass)
  for (int i = 0; i < R.np; i++)
    if (rr.pred_runs[i]) return false;  // an undecided dictionary leaf
  uint64_t sum_runs = 0;
  for (int k = 0; k < R.nk; k++) sum_runs += rr.n_runs[k];
  std::array<ChunkHost*, kRunsAggs> sums{};
  for (int a = 0; a < R.na; a++) {
    sums[size_t(a)] = rc.cols.ch[R.rd.agg_col[a]];
    if (!sums[size_t(a)] || sums[size_t(a)]->phys != PT_INT64) return false;
  }
  if (uint64_t(rr.n_rows) < kPrefixRunRows * sum_runs) return false;
  PrefixRg pr{};
  pr.n_rows = rr.n_rows;
  for (int k = 0; k < R.nk; k++) {  // (the directories are read by the plan's build step, not by an Execute)
    pr.runs[k] = rr.runs[k];
    pr.seeds[k] = rr.seeds[k];
    pr.n_runs[k] = rr.n_runs[k];
  }
  const uint32_t win = runs_prefix_window_rows(rr.n_rows, uint32_t(sum_runs));
  uint32_t n_win = 0;
  for (uint32_t r0 = 0; r0 < rr.n_rows; r0 += win, n_win++)
    P.wins.push_back(PrefixWin{uint32_t(P.rgs.size()), r0, std::min(win, rr.n_rows - r0), 0u});
  P.seg_bound += sum_runs + n_win;
  P.all_rows += rr.n_rows;
  // a Sum input is read at the segment boundaries, not row by row (PrefixBuilt counts those reads)
  uint32_t n_sums = 0;
  for (int a = 0; a < R.na; a++) {
    bool first = true;
    for (int a2 = 0; a2 < a; a2++) first = first && sums[size_t(a2)] != sums[size_t(a)];
    if (first) {
      st.algorithmic_bytes -= sums[size_t(a)]->stored_bytes;
      n_sums++;
    }
  }
  if (P.rgs.empty()) P.n_sums = n_sums;
  P.rgs.push_back(pr);
  P.sums.push_back(sums);
  P.parts.push_back(rc.cols.part);
  return true;
}

// Layout of both run kernels: the frame-of-reference and prefix-sum images (one batch over every staged int64 column
// and every Sum input of the prefix path of every part), then the tile rows and stage layout of k_runs_tma.
int32_t runs_layout(fgpu_ctx* ctx, const Compiled& c, const Switches& w, RunsPlan& R, PrefixPlan& P, fgpu_stats& st) {
  {
    std::set<std::pair<Part*, std::string>> seen, pseen;
    std::vector<std::pair<Part*, std::string>> want, want_prefix;
    for (const RunsRgCols& rc : R.cols)
      for (uint32_t i = 0; i < R.rd.n_cols; i++)
        if (rc.ch[i] && rc.ch[i]->phys == PT_INT64 && seen.emplace(rc.part, c.slot_names[size_t(R.col_slot[i])]).second)
          want.emplace_back(rc.part, c.slot_names[size_t(R.col_slot[i])]);
    for (size_t k = 0; k < P.rgs.size(); k++)
      for (int a = 0; a < R.na; a++)
        if (pseen.emplace(P.parts[k], c.slot_names[size_t(R.agg_slot[a])]).second) want_prefix.emplace_back(P.parts[k], c.slot_names[size_t(R.agg_slot[a])]);
    if (!want.empty() || !want_prefix.empty())
      if (int32_t rc = ensure_narrow(ctx, want, want_prefix)) return rc;
    for (size_t k = 0; k < P.rgs.size(); k++)
      for (int a = 0; a < R.na; a++) {
        P.rgs[k].pre[a] = P.sums[k][size_t(a)]->prefix;
        if (!P.rgs[k].pre[a]) return fail(FGPU_ERR_INVALID, "prefix-sum image missing for column " + c.slot_names[size_t(R.agg_slot[a])]);
      }
  }
  if (!P.rgs.empty()) {
    PrefixBuildDesc& bd = P.bd;
    bd.n_win = uint32_t(P.wins.size());
    bd.nk = uint32_t(R.nk);
    for (int k = 0; k < R.nk; k++) bd.stride[k] = R.rd.stride[k];
  }
  if (R.rgs.empty()) return FGPU_OK;
  RunsDesc& rd = R.rd;
  rd.n_rg = uint32_t(R.rgs.size());
  // every row group is cut into tiles of about tile_bytes of staged column data; the launch's tile table {row group,
  // first row} is dealt to the CTAs in chunks of consecutive entries
  const uint32_t tile_bytes = uint32_t(w.rt_tile) * 8u;  // (rows of 8 bytes)
  uint32_t tiles_rt = 0, gidx = 0, col_region = 0, max_tile = 1024;
  uint64_t total = 0;
  for (const RunsRg& r : R.rgs) total += r.n_rows;
  // small launches: at least one tile per resident CTA (three per SM), or the grid is not filled
  const uint32_t fill_rows = uint32_t(std::min<uint64_t>(1u << 20, std::max<uint64_t>(1024, (total / (uint64_t(ctx->sm_count) * 3)) & ~uint64_t(1023))));
  for (size_t k = 0; k < R.rgs.size(); k++) {
    RunsRg& r = R.rgs[k];
    uint32_t row_bytes = 0, max_runs = 0;
    for (uint32_t i = 0; i < rd.n_cols; i++) {
      const ChunkHost* ch = R.cols[k].ch[i];
      r.cl[i] = RunsCol{0, 3, 0};
      if (ch && ch->narrow) {
        r.col[i] = ch->narrow;
        r.cl[i].lg = ch->narrow_w == 1 ? 0 : (ch->narrow_w == 2 ? 1 : 2);
        r.cl[i].base = ch->narrow_base;
        st.algorithmic_bytes = st.algorithmic_bytes - ch->stored_bytes + uint64_t(r.n_rows) * ch->narrow_w;
      }
      if (r.col[i]) row_bytes += 1u << r.cl[i].lg;
    }
    for (int i = 0; i < R.nk; i++) max_runs = std::max(max_runs, r.n_runs[i]);
    for (int i = 0; i < R.np; i++)
      if (r.pred_runs[i]) max_runs = std::max(max_runs, r.pred_n_runs[i]);
    r.tile_rows = std::min(runs_tma_tile_rows(tile_bytes, row_bytes, r.n_rows, max_runs), fill_rows);
    int first = -1;
    uint32_t off = 0;
    for (uint32_t i = 0; i < rd.n_cols; i++) {
      if (!r.col[i]) continue;
      if (first < 0) first = int(i);
      r.cl[i].soff = off;
      off += ((r.tile_rows << r.cl[i].lg) + 127u) & ~127u;
    }
    for (uint32_t i = 0; i < rd.n_cols && first >= 0; i++)  // a column that is not staged reads a staged one
      if (!r.col[i]) r.cl[i] = r.cl[first];
    col_region = std::max(col_region, off);
    max_tile = std::max(max_tile, r.tile_rows);
    for (uint32_t r0 = 0; r0 < r.n_rows; r0 += r.tile_rows) {
      R.first_span.push_back(gidx);
      R.first_span.push_back(r0);
      tiles_rt++;
    }
    gidx++;
  }
  runs_tma_plan(rd, R.nk + R.np, max_tile, col_region, w.rt_stages, w.rt_warps, w.rt_span);
  rd.n_spans = tiles_rt;
  return FGPU_OK;
}

// The plan's segment table [seg_off | seg | build scratch] in sbuf, built behind the upload (count, scan, scatter),
// and the k_runs_prefix launch that reads it.  The build's segment count comes back to the page-locked word *count.
int32_t prefix_build(fgpu_ctx* ctx, const PrefixPlan& P, const RunsPlan& R, const QueryDesc& qd, DevBuf& sbuf, uint32_t* count, PrefixDesc* pd,
                     PrefixBuilt* pb, fgpu_stats& st) {
  // k_runs_prefix stores every cell of the table in place of k_table_init: only right when the table is dense and
  // every stored aggregate is Sum(int64) (identity 0), which prefix_query and runs_query let through
  if (qd.table_mode != TM_DENSE) return fail(FGPU_ERR_INVALID, "prefix path planned for a hash-mode table");
  for (int a = 0; a < qd.n_aggs; a++)
    if (qd.aggs[a].func != FGPU_AGG_COUNT && (qd.aggs[a].func != FGPU_AGG_SUM || qd.aggs[a].is_float))
      return fail(FGPU_ERR_INVALID, "prefix path planned for a table with an aggregate other than Sum(int64)");
  cudaStream_t s = ctx->stream;
  const uint32_t n_slots = uint32_t(qd.table_slots);
  const size_t off_bytes = HostImage::align16(size_t(n_slots + 1) * 4), seg_bytes = HostImage::align16(P.seg_bound * sizeof(PrefixSeg));
  CUDA_TRY(sbuf.alloc(off_bytes + seg_bytes + prefix_build_scratch_bytes(n_slots), s));
  uint8_t* sb = static_cast<uint8_t*>(sbuf.p);
  const uint32_t* seg_off = reinterpret_cast<const uint32_t*>(sb);
  PrefixBuildDesc bd = P.bd;
  bd.seg = reinterpret_cast<PrefixSeg*>(sb + off_bytes);
  CUDA_TRY(launch_prefix_build(bd, n_slots, reinterpret_cast<uint32_t*>(sb), sb + off_bytes + seg_bytes, ctx->sm_count, s));
  CUDA_TRY(cudaMemcpyAsync(count, seg_off + n_slots, 4, cudaMemcpyDeviceToHost, s));
  pb->count = count;
  pb->per_seg = sizeof(PrefixSeg) + 16 * uint64_t(P.n_sums);
  pb->launches = 3;  // count, scan (as one), scatter
  st.algorithmic_bytes += uint64_t(n_slots + 1) * 4;  // seg_off
  pd->n_slots = n_slots;
  pd->na = uint32_t(R.na);
  // lanes per slot: about one segment each up to a warp; a CTA per slot for lists of several hundred
  const uint64_t per_slot = (P.seg_bound + n_slots - 1) / n_slots;
  while (pd->group_log2 < 5 && (uint64_t(1) << pd->group_log2) < per_slot) pd->group_log2++;
  if (per_slot >= 256) pd->group_log2 = 8;
  pd->all_rows = P.all_rows;
  pd->rgs = bd.rgs;
  pd->seg_off = seg_off;
  pd->seg = bd.seg;
  bind_target(*pd, qd, R.agg_index, R.na);
  return FGPU_OK;
}

// ---- tile aggregate (tile_agg.cu) ----
// Row groups the sorted-run kernel does not take (bit-packed / short-run / nullable keys, L0 records) go to the
// tile-aggregate kernel when the plan is a conjunction of range + dictionary leaves over a dense table with plain
// aggregate inputs.
struct TilePlan {
  TileAggDesc td{};
  std::vector<TileAggRg> rgs;
  std::vector<uint32_t> first_tile;
  int plain_slot[kTaPlain] = {0}, code_slot[kTaCodes] = {0};
  uint32_t code_wmax[kTaCodes] = {0};
  int leaf_q[kTaLeaves] = {0}, pred_q[kTaPreds] = {0}, agg_index[kTaAggs] = {0};
  bool agg_bounded = true;  // every int64 Sum input of every row group has statistics inside [0, 2^32)
  uint64_t agg_max = 0;     // the largest of those chunk maxima
  size_t o_rgs = 0, o_first = 0;
  void place(HostImage& img) {
    o_rgs = img.add(rgs);
    o_first = img.add(first_tile);
  }
  void bind(uint8_t* block, const uint8_t* lut, const QueryDesc& qd, ScanLaunch& L) {
    lut_rebase(rgs, lut);
    L.tile = !rgs.empty();
    L.td = td;
    L.td.rgs = dev_at<const TileAggRg>(block, o_rgs);
    L.td.rg_first_tile = dev_at<const uint32_t>(block, o_first);
    bind_target(L.td, qd, agg_index, int(td.na));
  }
  uint32_t launches() const { return rgs.empty() ? 0 : 1; }  // k_tile_agg
};

bool tile_query(const Compiled& c, const QueryDesc& qd, const Switches& w, TilePlan* T) {
  if (w.no_tile || c.has_bool_keys() || c.has_unique() || qd.table_mode != TM_DENSE || (qd.n_filter_prog != 0 && qd.filter_kind != FK_AND) || qd.n_keys > kTaKeys)
    return false;
  TileAggDesc& td = T->td;
  auto plain_of = [&](int slot) { return find_or_add(T->plain_slot, &td.n_plain, kTaPlain, slot); };
  auto code_of = [&](int slot) { return find_or_add(T->code_slot, &td.n_codes, kTaCodes, slot); };
  for (int l = 0; l < qd.n_leaves; l++) {
    const LeafDesc& ld = qd.leaves[l];
    if (ld.slot == 0xff) continue;  // column absent from every row group: ALL / NONE per row group, nothing to evaluate
    if (qd.slot_type[ld.slot] == ST_DICT) {
      const int cc = code_of(ld.slot);
      if (td.np >= uint32_t(kTaPreds) || cc < 0) return false;
      T->pred_q[td.np] = l;
      td.pred_code[td.np++] = uint32_t(cc);
    } else {
      const int pp = plain_of(ld.slot);
      if (c.leaves[size_t(l)].null_literal || td.nl >= uint32_t(kTaLeaves) || pp < 0) return false;
      T->leaf_q[td.nl] = l;
      td.leaf_plain[td.nl] = uint32_t(pp);
      td.leaf_flags[td.nl++] = (ld.cmp_float ? 1u : 0u) | (qd.slot_type[ld.slot] == ST_F64 ? 2u : 0u) | (ld.neg ? 4u : 0u);
    }
  }
  for (int k = 0; k < qd.n_keys; k++) {
    const int cc = code_of(qd.keys[k].slot);
    if (qd.keys[k].is_int64 || cc < 0) return false;
    td.key_code[td.nk] = uint32_t(cc);
    td.key_stride[td.nk++] = qd.keys[k].dense_stride;
  }
  for (int a = 0; a < qd.n_aggs; a++) {
    const AggDesc& ad = qd.aggs[a];
    if (ad.func == FGPU_AGG_COUNT) continue;
    const bool simple = ad.prog_len == 1 && qd.prog[ad.prog_off].op == PO_LOAD;
    const int pp = simple ? plain_of(qd.prog[ad.prog_off].slot) : -1;
    if ((ad.func != FGPU_AGG_SUM && ad.func != FGPU_AGG_MIN && ad.func != FGPU_AGG_MAX) || td.na >= uint32_t(kTaAggs) || pp < 0) return false;
    T->agg_index[td.na] = a;
    td.agg_plain[td.na] = uint32_t(pp);
    td.cell64[td.na] = (ad.func == FGPU_AGG_SUM && !ad.is_float) ? 0u : 1u;
    td.agg_func[td.na++] = uint32_t(ad.func) | (ad.is_float ? 0x100u : 0u);
  }
  return true;
}

// *took: the kernel took the row group.  A row group where a leaf selects nothing is taken and dropped: under the
// conjunction no row of it passes.
int32_t tile_admit(TilePlan& T, fgpu_ctx* ctx, const Compiled& c, const QueryDesc& qd, const VisibleRG& v, const ChunkDesc* chunks, const LeafRt* lrt,
                   bool* took) {
  *took = false;
  const RowGroupHost& rg = *v.rg;
  if (rg.n_rows == 0) return FGPU_OK;
  const TileAggDesc& td = T.td;
  bool none = false;
  for (int l = 0; l < qd.n_leaves; l++)
    if (lrt[l].mode == LM_NONE) none = true;
  TileAggRg tr{};
  tr.n_rows = rg.n_rows;
  bool plain_needed[kTaPlain] = {false};
  for (uint32_t i = 0; i < td.nl; i++) {
    const int ql = T.leaf_q[i];
    const LeafDesc& ld = qd.leaves[ql];
    if (lrt[ql].mode == LM_ALL) { tr.leaf_skip[i] = 1; continue; }
    plain_needed[td.leaf_plain[i]] = true;
    if (ld.cmp_float) { std::memcpy(&tr.lo[i], &ld.lo_f, 8); std::memcpy(&tr.hi[i], &ld.hi_f, 8); }
    else { tr.lo[i] = ld.lo_i; tr.hi[i] = ld.hi_i; }
  }
  for (uint32_t i = 0; i < td.na; i++) plain_needed[td.agg_plain[i]] = true;
  for (uint32_t i = 0; i < td.n_plain && !none; i++) {
    const ChunkDesc& d = chunks[T.plain_slot[i]];
    tr.plain[i] = nullptr;
    if (!plain_needed[i]) continue;
    if (d.kind != CK_PLAIN64 || d.has_nulls) return FGPU_OK;
    tr.plain[i] = d.values;
  }
  bool code_needed[kTaCodes] = {false};
  for (uint32_t i = 0; i < td.np; i++) {
    const int ql = T.pred_q[i];
    const LeafRt& rt = lrt[ql];
    tr.pred_lut[i] = nullptr;
    if (rt.mode != LM_EVAL) continue;  // decided: passes (a NONE row group is dropped as a whole)
    code_needed[td.pred_code[i]] = true;
    tr.pred_lut[i] = lut_ref(c.leaves[size_t(ql)].lut_off);
    T.td.pred_null[i] = rt.null_result;
  }
  for (uint32_t i = 0; i < td.nk; i++) code_needed[td.key_code[i]] = true;
  for (uint32_t i = 0; i < td.n_codes && !none; i++) {
    const ChunkDesc& d = chunks[T.code_slot[i]];
    tr.codes[i] = nullptr;
    if (!code_needed[i] || d.kind == CK_ABSENT) continue;  // absent column: NULL for every row
    if (d.kind != CK_DICT_STR) return FGPU_OK;
    const std::string& name = c.slot_names[size_t(T.code_slot[i])];
    if (int32_t rc = ensure_flat(ctx, v.part, name)) return rc;
    const ChunkHost& ch = rg.cols.at(name);
    if (!ch.flat) return FGPU_OK;
    tr.codes[i] = ch.flat;
    tr.code_w[i] = ch.flat_w;
    tr.code_bias[i] = ch.flat_bias;
    T.code_wmax[i] = std::max<uint32_t>(T.code_wmax[i], ch.flat_w);
  }
  *took = true;
  if (none) return FGPU_OK;
  for (uint32_t i = 0; i < td.na; i++) {  // bounds of the int64 Sum inputs (see TileAggDesc::sums_fit32)
    if (td.cell64[i]) continue;
    const ChunkHost& ch = rg.cols.at(c.slot_names[size_t(T.plain_slot[td.agg_plain[i]])]);
    if (!ch.has_minmax || ch.phys != PT_INT64 || ch.min_bits < 0 || ch.max_bits > 0xffffffffll) T.agg_bounded = false;
    else T.agg_max = std::max<uint64_t>(T.agg_max, uint64_t(ch.max_bits));
  }
  T.rgs.push_back(tr);
  return FGPU_OK;
}

// Tile size, ring depth and the shared-memory table; the chunk of tiles a CTA takes at a time.
int32_t tile_layout(TilePlan& T, const QueryDesc& qd, const Switches& w, int sm_count) {
  TileAggDesc& td = T.td;
  td.n_rg = uint32_t(T.rgs.size());
  td.table_slots = qd.table_slots;
  // replicas of small tables: same-address CAS on 64-bit cells serialises, 32 lanes on 17 slots
  uint32_t rl = 0;
  while (rl < 5 && (uint64_t(qd.table_slots) << (rl + 1)) <= 2048) rl++;
  td.rep_log2 = rl;
  const uint64_t cells = uint64_t(qd.table_slots) << rl;
  uint64_t tb = (cells * 4 + 7) & ~uint64_t(7);
  for (uint32_t a = 0; a < td.na; a++) {
    td.cell_off[a] = uint32_t(tb);
    tb += (cells * (td.cell64[a] ? 8 : 4) + 7) & ~uint64_t(7);
  }
  const uint64_t kSmemMax = 227 * 1024;
  // tile rows: multiples of the rows the consumer threads take per turn (kTaConsumerWarps * 32 lanes * 4 rows)
  const int cand[10][2] = {{6144, 3}, {3072, 4}, {3072, 3}, {6144, 2}, {3072, 2}, {1536, 4}, {1536, 3}, {1536, 2}, {768, 3}, {768, 2}};
  auto slot_bytes_for = [&](uint32_t rows) {
    uint64_t off = 0;
    for (uint32_t i = 0; i < td.n_plain; i++) { td.plain_off[i] = uint32_t(off); off += uint64_t(rows) * 8; }
    for (uint32_t i = 0; i < td.n_codes; i++) {
      td.code_off[i] = uint32_t(off);
      off += (uint64_t(rows) * std::max<uint32_t>(T.code_wmax[i], 8) / 8 + 127) & ~uint64_t(127);
    }
    return std::max<uint64_t>(off, 128);
  };
  bool fits = false;
  for (int smem_table = tb < kSmemMax && !w.ta_global ? 1 : 0; smem_table >= 0 && !fits; smem_table--) {
    for (const auto& cs : cand) {
      if ((w.ta_tile && cs[0] != w.ta_tile) || (w.ta_stages && cs[1] != w.ta_stages)) continue;
      const uint64_t sb = slot_bytes_for(uint32_t(cs[0]));
      const uint64_t total = 128 + uint64_t(cs[1]) * (256 + sb) + (smem_table ? tb : 0);
      if (total > kSmemMax) continue;
      td.tile_rows = uint32_t(cs[0]);
      td.n_stages = uint32_t(cs[1]);
      td.slot_bytes = uint32_t(sb);
      td.smem_table = uint32_t(smem_table);
      fits = true;
      break;
    }
  }
  if (!fits) return fail(FGPU_ERR_UNSUPPORTED, "tile aggregate: the projected columns do not fit the shared-memory ring");
  td.table_bytes = uint32_t(td.smem_table ? tb : 0);
  uint32_t t = 0;
  for (const TileAggRg& r : T.rgs) {
    T.first_tile.push_back(t);
    t += (r.n_rows + td.tile_rows - 1) / td.tile_rows;
  }
  T.first_tile.push_back(t);
  td.n_tiles = t;
  td.chunk_tiles = std::max<uint32_t>(1, t / (uint32_t(sm_count) * 4));  // ~4 turns per CTA: a CTA stays inside one row group for a whole chunk
  // (the override comes first: the 32-bit Sum bound below depends on the chunk length the launch uses)
  if (w.ta_chunk) td.chunk_tiles = uint32_t(w.ta_chunk);
  td.keys8 = 1;
  for (uint32_t i = 0; i < td.nk; i++)
    if (T.code_wmax[td.key_code[i]] > 8) td.keys8 = 0;
  {  // can a Sum leave 32 bits inside one CTA?  rows per CTA <= its share of the tiles (+ one chunk), all in one slot
    const uint64_t grid = uint64_t(std::max(1, sm_count));
    const uint64_t rows_per_cta = std::min<uint64_t>(uint64_t(t), uint64_t(t) / grid + 2 * uint64_t(td.chunk_tiles) + 1) * td.tile_rows;
    // agg_max * rows_per_cta <= 2^32 - 1, without the product (a large chunk override would overflow it)
    td.sums_fit32 = (T.agg_bounded && !w.ta_carry && (T.agg_max == 0 || rows_per_cta <= 0xffffffffull / T.agg_max)) ? 1u : 0u;
  }
  return FGPU_OK;
}

// ---- filter-only plans over PLAIN columns: ordered take (take_rows.cu) instead of k_rows ----
struct TakePlan {
  TakeDesc td{};
  std::vector<TakeRg> rgs;
  std::vector<uint32_t> first_span;
  int range[kTakeLeaves] = {0}, pred[kTakePreds] = {0};  // range leaves (PLAIN int64 columns) and dictionary leaves (flat
  int n_range = 0, n_pred = 0;                           // codes + result byte per dictionary id) of the plan
  size_t o_rgs = 0, o_span = 0, o_count = 0;
  void place(HostImage& img) {
    o_rgs = img.add(rgs);
    o_span = img.add(first_span);
    o_count = img.add(nullptr, (size_t(td.n_spans) + 1) * 8);
  }
  void bind(uint8_t* block, const uint8_t* lut, const QueryDesc& qd) {
    lut_rebase(rgs, lut);
    td.rgs = dev_at<const TakeRg>(block, o_rgs);
    td.rg_first_span = dev_at<const uint32_t>(block, o_span);
    td.span_count = dev_at<unsigned long long>(block, o_count);
    td.total = qd.counters;
    for (int o = 0; o < qd.n_out; o++) td.out_data[o] = static_cast<long long*>(qd.out_data[o]);
  }
  uint32_t launches() const { return td.n_spans ? 3 : 0; }  // count per span, scan, ordered write
};

// general: row groups left with the general kernel (all of them unless pruning dropped some).
bool take_query(const Compiled& c, const QueryDesc& qd, const Switches& w, int general, TakePlan* P) {
  if (w.no_take || qd.n_out < 1 || qd.n_out > kTakeOut || qd.n_leaves > kTakeLeaves + kTakePreds || (qd.n_filter_prog != 0 && qd.filter_kind != FK_AND) ||
      general == 0)
    return false;
  for (int l = 0; l < qd.n_leaves; l++) {
    const LeafDesc& ld = qd.leaves[l];
    if (ld.slot == 0xff) return false;
    if (qd.slot_type[ld.slot] == ST_DICT) {
      if (P->n_pred >= kTakePreds || general != c.qd.n_rg) return false;
      P->pred[P->n_pred++] = l;
    } else if (ld.cmp_float || ld.neg || qd.slot_type[ld.slot] != ST_I64 || c.leaves[size_t(l)].null_literal || P->n_range >= kTakeLeaves) {
      return false;
    } else {
      P->range[P->n_range++] = l;
    }
  }
  for (int o = 0; o < qd.n_out; o++)
    if (qd.slot_type[qd.out_slot[o]] == ST_DICT) return false;
  return true;
}

// *ok: the take kernels can read row group g (rows plans: every row group is a general one, g == its index in c.rgs).
int32_t take_admit(TakePlan& P, fgpu_ctx* ctx, const Compiled& c, const QueryDesc& qd, int g, const GeneralTables& G, bool* ok) {
  *ok = false;
  const ChunkDesc* chunks = &G.chunks[size_t(g) * qd.n_slots];
  const LeafRt* lrt = &G.lrt[size_t(g) * qd.n_leaves];
  TakeRg tr{};
  tr.n_rows = G.rg_rows[size_t(g)];
  bool all = qd.n_leaves > 0;
  for (int l = 0; l < qd.n_leaves; l++) {
    if (lrt[l].mode == LM_NONE) return FGPU_OK;  // (only with pruning switched off)
    if (lrt[l].mode != LM_ALL) all = false;
  }
  tr.all_pass = all ? 1 : 0;
  for (int i = 0; i < P.n_range; i++) {
    const int l = P.range[i];
    const bool decided = lrt[l].mode == LM_ALL;
    tr.lo[i] = decided ? std::numeric_limits<int64_t>::min() : qd.leaves[l].lo_i;
    tr.hi[i] = decided ? std::numeric_limits<int64_t>::max() : qd.leaves[l].hi_i;
    tr.leaf_col[i] = nullptr;  // decided (or nothing to evaluate at all): the kernels skip the leaf
    if (all || decided) continue;
    const ChunkDesc& d = chunks[qd.leaves[l].slot];
    if (d.kind != CK_PLAIN64 || d.has_nulls) return FGPU_OK;
    tr.leaf_col[i] = d.values;
  }
  for (int i = 0; i < P.n_pred; i++) {
    const int l = P.pred[i];
    const LeafRt& rt = lrt[l];
    tr.pred_codes[i] = nullptr;
    if (all || rt.mode == LM_ALL) continue;
    const ChunkDesc& d = chunks[qd.leaves[l].slot];
    if (d.kind != CK_DICT_STR) return FGPU_OK;
    const std::string& name = c.slot_names[size_t(qd.leaves[l].slot)];
    if (int32_t rc = ensure_flat(ctx, c.rgs[size_t(g)].part, name)) return rc;
    const ChunkHost& ch = c.rgs[size_t(g)].rg->cols.at(name);
    if (!ch.flat) return FGPU_OK;
    tr.pred_codes[i] = ch.flat;
    tr.pred_w[i] = ch.flat_w;
    tr.pred_bias[i] = ch.flat_bias;
    tr.pred_null[i] = rt.null_result;
    tr.pred_lut[i] = lut_ref(c.leaves[size_t(l)].lut_off);
  }
  for (int o = 0; o < qd.n_out; o++) {
    const ChunkDesc& d = chunks[qd.out_slot[o]];
    if (d.kind != CK_PLAIN64 || d.has_nulls) return FGPU_OK;
    tr.out_col[o] = d.values;
  }
  P.rgs.push_back(tr);
  *ok = true;
  return FGPU_OK;
}

// Spans of span_blocks * 256 rows, about four per resident warp.
void take_layout(TakePlan& P, const QueryDesc& qd, int sm_count) {
  TakeDesc& td = P.td;
  const uint64_t warps = uint64_t(take_resident_warps(sm_count));
  uint64_t total = 0;
  for (const TakeRg& r : P.rgs) total += r.n_rows;
  uint64_t span_blocks = std::min<uint64_t>(64, std::max<uint64_t>(4, total / (warps * 4 * 256)));
  td.span_blocks = uint32_t(span_blocks);
  const uint64_t span_rows = span_blocks * 256;
  uint32_t spans = 0;
  for (const TakeRg& r : P.rgs) {
    P.first_span.push_back(spans);
    spans += uint32_t((uint64_t(r.n_rows) + span_rows - 1) / span_rows);
  }
  P.first_span.push_back(spans);
  td.n_spans = spans;
  td.n_rg = uint32_t(P.rgs.size());
  td.nl = uint32_t(P.n_range);
  td.np = uint32_t(P.n_pred);
  td.n_out = uint32_t(qd.n_out);
}

// The result's columns (see ResultShape), with the key dictionaries snapshotted now.
ResultShape result_shape(const QueryPlan& q, const Compiled& c) {
  ResultShape r;
  r.keys = c.keys;
  for (KeyOut& k : r.keys) {
    if (k.dict) {
      const uint32_t card = k.dict->cardinality();
      k.dict_snapshot.reserve(card);
      for (uint32_t i = 0; i < card; i++) k.dict_snapshot.push_back(k.dict->value(i));
      k.dict = nullptr;
    }
  }
  for (size_t a = 0, cell = 0; a < q.aggs.size(); a++) {
    r.agg_names.push_back(std::string(agg_string(q.aggs[a].func)) + "(" + q.expr_name(q.aggs[a].expr) + ")");
    // Count yields int64; Sum/Min/Max keep the input type (aggregate.go:734-950); Unique is int64 only
    r.agg_is_float.push_back(c.qd.aggs[cell].func != FGPU_AGG_COUNT && c.qd.aggs[cell].is_float);
    cell += c.qd.aggs[cell].unique ? 2 : 1;
  }
  return r;
}

// First Execute of a cached plan: the plan keeps the device state; the dense table comes back compacted by
// k_finalize_dense (see ExecCache).
int32_t keep_exec_cache(fgpu_ctx* ctx, const QueryPlan& q, Compiled& c, const QueryDesc& qd, fgpu_result* res, PhaseClock& pc,
                        const PrefixBuilt& pb) {
  cudaStream_t s = ctx->stream;
  fgpu_stats& st = res->stats;
  ExecCache& x = *c.exec;
  DenseOut& f = x.dout;
  f.table_slots = qd.table_slots;
  f.max_out = qd.table_slots;
  f.n_keys = uint32_t(qd.n_keys);
  f.n_aggs = uint32_t(qd.n_aggs);
  for (int k = 0; k < qd.n_keys; k++) {
    f.stride[k] = qd.keys[k].dense_stride;
    f.radix[k] = c.radix(k);
  }
  f.t_rows = qd.t_rows;
  for (int a = 0; a < kMaxAggs; a++) f.t_agg[a] = qd.t_agg[a];
  f.counters = qd.counters;
  {  // what the collective tail needs to fold partial tables itself (layout of table_layout())
    int pos = 0;
    for (int a = 0; a < qd.n_aggs; a++) {
      f.agg_func[a] = qd.aggs[a].func;
      f.agg_is_float[a] = qd.aggs[a].is_float;
      f.agg_unique[a] = qd.aggs[a].unique;
      f.agg_pos[a] = qd.aggs[a].func == FGPU_AGG_COUNT ? int8_t(-1) : int8_t(pos++);
    }
  }
  x.out_bytes = 256 + size_t(qd.n_keys) * ((size_t(f.max_out) * 4 + 7) & ~size_t(7)) + size_t(qd.n_aggs) * f.max_out * 8;
  CUDA_TRY(x.out.alloc(256, s));  // working header (k_finalize_dense leaves it zero)
  CUDA_TRY(cudaMemsetAsync(x.out.p, 0, 256, s));
  f.hdr = static_cast<uint32_t*>(x.out.p);
  f.out = nullptr;  // a page-locked block per Execute (cached_tail)
  x.pinned = PinnedBlock(ctx->pinned, x.out_bytes);
  if (!x.pinned) return fail(FGPU_ERR_OOM, "page-locked memory for the result image");
  if (!res->pending) {
    if (int32_t rc = cached_tail(ctx, x)) return rc;
  } else {
    CUDA_TRY(cudaMemcpyAsync(x.pinned.get() + 32, qd.counters, 32, cudaMemcpyDeviceToHost, s));  // (rows selected by this rank's scan)
  }
  if (int32_t rc = finish_scan(ctx, pc, st, /*total=*/true)) return rc;  // the host image stays valid until here
  st.h2d_bytes += c.h2d_bytes;
  const unsigned long long* cnts = reinterpret_cast<const unsigned long long*>(x.pinned.get() + 32);
  st.rows_selected = cnts[0];
  pb.account(st);
  x.qd = qd;
  x.shape = result_shape(q, c);
  for (const KeyOut& k : x.shape.keys) {  // small dictionaries are exported whole: the host then only copies index columns
    x.dict_template.push_back(!k.is_bool && k.dict_snapshot.size() <= 4096 ? dict_column(k.dict_snapshot, nullptr) : nullptr);
  }
  x.stats = st;  // what a cached Execute reports: no uploads, no compile, no segment-table build
  x.stats.kernel_launches -= pb.launches;
  x.stats.h2d_bytes = 0;
  x.stats.d2h_bytes = 0;
  x.stats.rows_selected = 0;
  x.ready = true;
  st.d2h_bytes += x.out_bytes;
  res->qd = qd;
  pc.mark("keep");
  pc.flush("scan");
  if (res->pending) {
    res->pending_cached = &x;
    return FGPU_OK;
  }
  return finalize_dense_host(res, x);
}

FinalizeDesc finalize_desc(const Compiled& c, const QueryDesc& qd) {
  FinalizeDesc fd{};
  fd.table_mode = qd.table_mode;
  fd.key_words = qd.key_words;
  fd.n_keys = qd.n_keys;
  fd.n_aggs = qd.n_aggs;
  fd.table_slots = qd.table_slots;
  for (int k = 0; k < qd.n_keys; k++) {
    fd.keys[k] = qd.keys[k];
    fd.dense_radix[k] = c.radix(k);
  }
  for (int a = 0; a < qd.n_aggs; a++) fd.agg_unique[a] = qd.aggs[a].unique;
  bind_finalize(&fd, qd);
  return fd;
}

// Rows plan: one output array per projected column (worst case every row is selected) + look-back state per tile.
int32_t alloc_rows_out(fgpu_ctx* ctx, uint64_t total_rows, uint32_t tiles, DevBuf& buf, QueryDesc* qd) {
  std::vector<size_t> out_off(size_t(qd->n_out)), valid_off(size_t(qd->n_out));
  size_t out_bytes = 0;
  auto al = [](size_t x) { return (x + 255) & ~size_t(255); };
  for (int o = 0; o < qd->n_out; o++) {
    bool dict = qd->slot_type[qd->out_slot[o]] == ST_DICT;
    out_off[size_t(o)] = out_bytes;
    out_bytes = al(out_bytes + size_t(total_rows) * (dict ? 4 : 8));
    valid_off[size_t(o)] = out_bytes;
    if (!dict) out_bytes = al(out_bytes + size_t(total_rows));
  }
  const size_t state_off = out_bytes;
  out_bytes = al(out_bytes + size_t(tiles) * 8);
  CUDA_TRY(buf.alloc(out_bytes, ctx->stream));
  uint8_t* ob = static_cast<uint8_t*>(buf.p);
  for (int o = 0; o < qd->n_out; o++) {
    qd->out_data[o] = ob + out_off[size_t(o)];
    qd->out_valid[o] = ob + valid_off[size_t(o)];
  }
  qd->tile_state = reinterpret_cast<unsigned long long*>(ob + state_off);
  return FGPU_OK;
}

// The query's compiled plan in q.plan_cache: the one it holds while the table epoch, the read transaction and the
// switches are those it was compiled for, a fresh one otherwise.
int32_t compiled_plan(fgpu_ctx* ctx, const QueryPlan& q, uint64_t tx, const Switches& w) {
  Table& plan_table = ctx->tables[q.table];
  if (plan_table.epoch == 0) plan_table.epoch = ++ctx->epoch_counter;
  if (q.plan_cache && q.cache_epoch == plan_table.epoch && q.cache_tx == tx && q.cache_env == w.key && !w.no_plan_cache) {
    static_cast<Compiled*>(q.plan_cache.get())->h2d_bytes = 0;  // nothing is uploaded by a cached plan
    return FGPU_OK;
  }
  std::shared_ptr<void> fresh(new Compiled(), [](void* p) { delete static_cast<Compiled*>(p); });
  int32_t rc = compile(ctx, q, tx, w, static_cast<Compiled*>(fresh.get()));
  q.plan_cache.reset();
  if (rc) return rc;
  q.plan_cache = std::move(fresh);
  q.cache_epoch = plan_table.epoch;
  q.cache_tx = tx;
  q.cache_env = w.key;
  return FGPU_OK;
}

// Row groups of the plan -> the general tables, or the sorted-run, prefix-sum or tile-aggregate plan that takes them.
int32_t route_row_groups(fgpu_ctx* ctx, const QueryPlan& q, Compiled& c, const QueryDesc& qd, const Switches& w, bool rows_plan, GeneralTables& G,
                         RunsPlan& R, PrefixPlan& P, TilePlan& T, fgpu_stats& st) {
  const int n_slots = qd.n_slots, n_leaves = qd.n_leaves;
  const uint32_t tile_len = rows_plan ? uint32_t(kTileRows) : uint32_t(qd.vl);  // rows plan: CTA tiles; scan: warp vectors
  const bool runs_q = !rows_plan && runs_query(c, qd, w, &R);
  const bool prefix_q = runs_q && prefix_query(c, R, w);
  const bool tile_q = !rows_plan && tile_query(c, qd, w, &T);
  for (int g0 = 0; g0 < qd.n_rg; g0++) {
    const size_t lut_mark = G.lut_fix.size();
    if (int32_t rc = describe_row_group(ctx, q, c, g0, G, st)) return rc;
    const VisibleRG& v = c.rgs[size_t(g0)];
    const ChunkDesc* row_chunks = &G.chunks[size_t(G.n) * n_slots];
    const LeafRt* row_lrt = &G.lrt[size_t(G.n) * n_leaves];
    bool took = false;
    RunsCand rc;
    if (runs_q && runs_admit(R, c, qd, v, row_chunks, row_lrt, &rc)) {
      if (!(prefix_q && prefix_admit(P, R, rc, st))) {
        R.rgs.push_back(rc.rr);
        R.cols.push_back(rc.cols);
      }
      took = true;
    } else if (tile_q) {
      if (int32_t e = tile_admit(T, ctx, c, qd, v, row_chunks, row_lrt, &took)) return e;
    }
    if (took) {  // slot G.n of the general tables is reused by the next row group
      G.lut_fix.resize(lut_mark);
      continue;
    }
    G.first_tile[size_t(G.n)] = G.tiles;
    G.rg_rows[size_t(G.n)] = v.rg->n_rows;
    G.tiles += (v.rg->n_rows + tile_len - 1) / tile_len;
    G.n++;
  }
  G.first_tile[size_t(G.n)] = G.tiles;
  return FGPU_OK;
}

// Plans and launches one Execute.  On success the result owns the device table (or, for a cached plan, the plan does).
// collective: 0 no exchange; 1 / 2: the first run of a plan pushes its partial table and leaves the result pending
// (the merge half is collective_end); a cached plan does what run_cached does for the mode.
int32_t run_scan(fgpu_ctx* ctx, const QueryPlan& q, uint64_t tx, fgpu_result* res, bool count_groups = false, bool cacheable = false,
                 int collective = 0) {
  PhaseClock pc;
  const Switches w = switches();
  if (int32_t rc = compiled_plan(ctx, q, tx, w)) return rc;
  Compiled& c = *static_cast<Compiled*>(q.plan_cache.get());
  if (cacheable && c.exec && c.exec->ready && !w.no_exec_cache) return run_cached(ctx, *c.exec, res, collective);
  c.exec.reset();
  for (LeafHost& lh : c.leaves) lh.lut_off = size_t(-1);  // per-Execute state of the plan
  for (LeafHost& lh : c.key_leaves) lh.lut_off = size_t(-1);
  pc.mark("compile");
  QueryDesc qd = c.qd;  // a copy: the plan in `c` may be reused by the next Execute
  const int n_rg = qd.n_rg;
  const bool rows_plan = q.kind == FGPU_PLAN_FILTER;
  fgpu_stats& st = res->stats;
  st.rows_scanned = c.total_rows;
  st.rows_touched = c.touched_rows == ~uint64_t(0) ? c.total_rows : c.touched_rows;
  st.row_groups = uint32_t(n_rg);
  st.row_groups_pruned = c.pruned_row_groups;

  // ---- where every row group goes ----
  GeneralTables G(n_rg, qd.n_slots, qd.n_leaves, int(c.key_leaves.size()));
  RunsPlan R;
  PrefixPlan P;
  TilePlan T;
  if (int32_t rc = route_row_groups(ctx, q, c, qd, w, rows_plan, G, R, P, T, st)) return rc;
  qd.n_rg = G.n;
  qd.n_tiles = G.tiles;
  if (int32_t rc = runs_layout(ctx, c, w, R, P, st)) return rc;
  if (!T.rgs.empty())
    if (int32_t rc = tile_layout(T, qd, w, ctx->sm_count)) return rc;
  TakePlan K;
  bool take_q = rows_plan && take_query(c, qd, w, G.n, &K);
  for (int g = 0; g < G.n && take_q; g++)
    if (int32_t rc = take_admit(K, ctx, c, qd, g, G, &take_q)) return rc;
  if (take_q) take_layout(K, qd, ctx->sm_count);

  // ---- device memory -----------------------------------------------------------------------
  // small dense tables of a re-executable query: persistent device state owned by the plan (ExecCache)
  const bool cache_mode = cacheable && !rows_plan && qd.table_mode == TM_DENSE && qd.table_slots <= 65536 && !w.no_exec_cache;
  if (cache_mode) c.exec.reset(new ExecCache());
  DevBuf& tbuf = cache_mode ? c.exec->table : res->table;
  DevBuf& abuf = cache_mode ? c.exec->aux : res->aux;
  size_t tbytes = 0;
  if (!rows_plan) {
    size_t off_aggs, off_tags, off_keys;
    tbytes = table_layout(qd, &off_aggs, &off_tags, &off_keys);
    CUDA_TRY(tbuf.alloc(tbytes + 128, ctx->stream));  // (+ counters in cache mode; slack for the 16-byte exchange copies)
    res->table_bytes = tbytes;
    bind_table(&qd, static_cast<uint8_t*>(tbuf.p));
  } else if (int32_t rc = alloc_rows_out(ctx, c.total_rows, G.tiles, tbuf, &qd)) {
    return rc;
  }

  // device block: [plans' tables | counters 64 B | group counter 16 B | QueryDesc]
  HostImage img;
  G.place(img, c);
  R.place(img);
  P.place(img);
  T.place(img);
  if (take_q) K.place(img);
  const size_t o_cnt = img.add(nullptr, 64 + 16);
  const size_t o_qd = img.add(&qd, sizeof(QueryDesc));
  const size_t aux_bytes = img.end;
  const size_t o_ret = HostImage::align16(aux_bytes);  // scratch only: counters + group count read back
  CUDA_TRY(abuf.alloc(aux_bytes, ctx->stream));
  uint8_t* aux = static_cast<uint8_t*>(abuf.p);
  qd.counters = cache_mode ? reinterpret_cast<unsigned long long*>(static_cast<uint8_t*>(tbuf.p) + tbytes)  // behind the table: one copy brings both back
                           : dev_at<unsigned long long>(aux, o_cnt);
  ScanLaunch L;
  const uint8_t* lut = G.bind(aux, qd);
  R.bind(aux, lut, qd, L);
  P.bind(aux, L);
  T.bind(aux, lut, qd, L);
  if (take_q) K.bind(aux, lut, qd);
  const QueryDesc* qdesc_dev = dev_at<const QueryDesc>(aux, o_qd);
  CUDA_TRY(ctx->ensure_scratch(o_ret + 128));
  std::memset(ctx->scratch, 0, o_ret + 128);
  img.copy_to(ctx->scratch);

  FinalizeDesc& fd = res->fd;
  fd = finalize_desc(c, qd);
  cudaStream_t s = ctx->stream;
  pc.mark("describe");
  CUDA_TRY(cudaEventRecord(ctx->ev[0], s));
  CUDA_TRY(cudaMemcpyAsync(aux, ctx->scratch, aux_bytes, cudaMemcpyHostToDevice, s));
  PrefixBuilt pb;
  if (rows_plan) {
    CUDA_TRY(cudaMemsetAsync(qd.tile_state, 0, size_t(G.tiles) * 8, s));
    CUDA_TRY(cudaEventRecord(ctx->ev[1], s));
    if (take_q) {
      CUDA_TRY(launch_take(K.td, ctx->sm_count, s));
      res->rows_no_nulls = true;
    } else {
      CUDA_TRY(launch_rows(qdesc_dev, qd, ctx->sm_count, s));
    }
    CUDA_TRY(cudaEventRecord(ctx->ev[2], s));
  } else {
    if (L.prefix) {
      uint32_t* count = reinterpret_cast<uint32_t*>(ctx->scratch + o_ret + 96);
      if (int32_t rc = prefix_build(ctx, P, R, qd, cache_mode ? c.exec->segs : res->segs, count, &L.pd, &pb, st)) return rc;
    }
    if (int32_t rc = launch_aggregate_scan(ctx, qd, qdesc_dev, L)) return rc;
    st.row_groups_runs += uint32_t(R.rgs.size() + P.rgs.size());
    st.row_groups_prefix += uint32_t(P.rgs.size());
    st.row_groups_tiles += uint32_t(T.rgs.size());
  }
  // k_table_init unless k_runs_prefix stores the table; k_finalize_dense of a kept plan, or the group count behind the scan
  count_groups = count_groups && !rows_plan && !cache_mode && !collective;  // (a collective Execute's table is not final yet)
  st.kernel_launches += (rows_plan || L.prefix ? 0 : 1) + (take_q ? K.launches() : G.launches()) + R.launches() + P.launches() + pb.launches +
                        T.launches() + (cache_mode ? 1 : 0) + (count_groups ? 1 : 0);
  st.h2d_bytes += aux_bytes + sizeof(QueryDesc);
  unsigned long long* counters = reinterpret_cast<unsigned long long*>(ctx->scratch + o_ret);
  res->cnt_ptr = reinterpret_cast<unsigned int*>(qd.counters + 8);  // 16 bytes behind the counters, zeroed by the upload / the table init
  if (collective) {
    if (rows_plan) return fail(FGPU_ERR_INVALID, "rows plans have no partial table: execute them per rank");
    if (int32_t rc = comm_push(ctx, tbuf.p, tbytes, &res->pending_seq, &res->pending_bytes)) return rc;
    res->pending = true;
    res->plan_keep = q.plan_cache;
  }
  if (cache_mode) {
    ExecCache& x = *c.exec;
    x.table_bytes = tbytes;
    x.qdesc_dev = qdesc_dev;
    x.launch = L;
    return keep_exec_cache(ctx, q, c, qd, res, pc, pb);
  }
  if (count_groups) {  // count the result rows behind the scan: one host round trip less
    CUDA_TRY(launch_count_groups(fd, res->cnt_ptr, s));
    res->groups_known = true;
  }
  CUDA_TRY(cudaMemcpyAsync(counters, qd.counters, 64 + 16, cudaMemcpyDeviceToHost, s));
  if (int32_t rc = finish_scan(ctx, pc, st, /*total=*/false)) return rc;  // the host image / counters stay valid until here
  st.h2d_bytes += c.h2d_bytes;
  st.rows_selected = counters[0];
  pb.account(st);
  if (res->groups_known) res->n_groups = static_cast<unsigned int>(counters[8] & 0xffffffffull);
  st.d2h_bytes += 64;
  if (counters[1]) return fail(FGPU_ERR_UNSUPPORTED, "aggregate hash table overflow (more groups than the sized capacity)");
  if (int32_t rc = comm_check(counters[3])) return rc;

  // keep what finalize / merge need
  res->qd = qd;
  res->rows_plan = rows_plan;
  res->shape = result_shape(q, c);
  pc.mark("keep");
  pc.flush("scan");
  return FGPU_OK;
}

// Compacted result image in page-locked memory -> one Arrow record (finishAggregate, aggregate.go:543-633): the
// device already produced dictionary indices and aggregate values per result row (k_finalize_dense); the host copies.
int32_t finalize_dense_host(fgpu_result* res, ExecCache& x) {
  PhaseClock pc;
  const QueryDesc& qd = x.qd;
  uint8_t* img = x.pinned.get();
  const uint32_t* hdr = reinterpret_cast<const uint32_t*>(img);
  const size_t G = std::min<size_t>(hdr[0], x.dout.max_out);
  res->stats.groups = G;
  const int nk = qd.n_keys, na = qd.n_aggs;
  const size_t key_bytes = (size_t(x.dout.max_out) * 4 + 7) & ~size_t(7);
  std::vector<OwnedColumn> cols;
  cols.reserve(size_t(nk + na));
  // the columns of the record are slices of the page-locked block the kernel wrote: the record takes the block (the next
  // Execute takes another one), and it goes back to the pool when the consumer has released every array
  std::shared_ptr<void> keep;
  if (G > 0) keep = std::move(x.pinned).keep();
  for (int k = 0; k < nk; k++) {
    const KeyOut& ko = x.shape.keys[size_t(k)];
    uint32_t* idx = reinterpret_cast<uint32_t*>(img + 256 + size_t(k) * key_bytes);
    OwnedColumn col;
    col.name = ko.name;
    col.length = int64_t(G);
    if (G > 0) {
      col.ext = reinterpret_cast<const uint8_t*>(idx);
      col.ext_keep = keep;
    }
    if (ko.is_bool) {  // bits packed in place
      bool_key_column(col, idx, G);
      cols.push_back(std::move(col));
      continue;
    }
    // ids re-indexed in place; hdr[16 + k]: the kernel wrote a NULL key
    const OwnedColumn* whole = x.dict_template[size_t(k)].get();
    dict_key_column(col, idx, G, idx, ko.dict_snapshot, whole ? KeyDict::kWhole : KeyDict::kUsed, whole, hdr[16 + k] != 0);
    cols.push_back(std::move(col));
  }
  const uint8_t* aggs = img + 256 + size_t(nk) * key_bytes;
  for (int a = 0, o = 0; a < na; a++) {
    if (qd.aggs[a].unique == UC_HI) continue;  // the validity of the Unique before it
    OwnedColumn col;
    col.name = x.shape.agg_names[size_t(o)];
    col.format = x.shape.agg_is_float[size_t(o++)] ? "g" : "l";
    col.length = int64_t(G);
    if (G > 0) {
      col.ext = aggs + size_t(a) * x.dout.max_out * 8;
      col.ext_keep = keep;
    }
    if (qd.aggs[a].unique == UC_LO) validity_from_bytes(col, aggs + size_t(a + 1) * x.dout.max_out * 8, G);
    cols.push_back(std::move(col));
  }
  res->stats.algorithmic_bytes += (size_t(nk) + size_t(na)) * G * 8;
  res->finish(std::move(cols), G);
  pc.mark("arrow");
  pc.flush("finalize-host");
  return FGPU_OK;
}

// Table -> host columns -> one Arrow record.
// Rows plan: selected rows of the projected columns -> one Arrow record (filter.go:276-323 + Projection).
int32_t finalize_rows(fgpu_ctx* ctx, fgpu_result* res) {
  cudaStream_t s = ctx->stream;
  const QueryDesc& qd = res->qd;
  const size_t R = size_t(res->stats.rows_selected);
  res->stats.groups = R;
  // Every projected column comes back into a page-locked block of the context's pool with ONE copy each and ONE
  // synchronisation for all of them; the block itself becomes the Arrow buffer (it returns to the pool when the
  // consumer releases the array), so a large selection costs its PCIe transfer and nothing else.
  std::vector<PinnedBlock> data(size_t(qd.n_out)), valid(size_t(qd.n_out));
  for (int o = 0; o < qd.n_out && R; o++) {
    const bool dict = !res->shape.keys[size_t(o)].is_int64;
    const size_t bytes = R * (dict ? 4 : 8);
    data[size_t(o)] = PinnedBlock(ctx->pinned, bytes);
    if (!data[size_t(o)]) return fail(FGPU_ERR_OOM, "page-locked memory for the result rows");
    CUDA_TRY(cudaMemcpyAsync(data[size_t(o)].get(), qd.out_data[o], bytes, cudaMemcpyDeviceToHost, s));
    res->stats.d2h_bytes += bytes;
    if (!dict && !res->rows_no_nulls) {
      valid[size_t(o)] = PinnedBlock(ctx->pinned, R);
      if (!valid[size_t(o)]) return fail(FGPU_ERR_OOM, "page-locked memory for the result rows");
      CUDA_TRY(cudaMemcpyAsync(valid[size_t(o)].get(), qd.out_valid[o], R, cudaMemcpyDeviceToHost, s));
      res->stats.d2h_bytes += R;
    }
  }
  CUDA_TRY(cudaEventRecord(ctx->ev[3], s));
  CUDA_TRY(cudaStreamSynchronize(s));
  float ms = 0;
  cudaEventElapsedTime(&ms, ctx->ev[0], ctx->ev[3]);
  res->stats.total_device_ms = ms;
  std::vector<OwnedColumn> cols;
  for (int o = 0; o < qd.n_out; o++) {
    const KeyOut& ko = res->shape.keys[size_t(o)];
    uint8_t* p = data[size_t(o)].get();
    OwnedColumn col;
    col.name = ko.name;
    col.length = int64_t(R);
    if (!ko.is_int64) {  // dictionary ids (-1 = NULL), re-indexed in place
      dict_key_column(col, reinterpret_cast<const int32_t*>(p), R, reinterpret_cast<uint32_t*>(p), ko.dict_snapshot, KeyDict::kUsed);
    } else {
      col.format = ko.is_float ? "g" : "l";
      if (valid[size_t(o)]) validity_from_bytes(col, valid[size_t(o)].get(), R);
    }
    if (R) {
      col.ext = p;
      col.ext_keep = std::move(data[size_t(o)]).keep();
    }
    res->stats.algorithmic_bytes += R * (ko.is_int64 ? 8 : 4);
    cols.push_back(std::move(col));
  }
  res->finish(std::move(cols), R);
  res->table.reset();
  res->aux.reset();
  return FGPU_OK;
}

int32_t finalize_result(fgpu_ctx* ctx, fgpu_result* res) {
  if (res->rows_plan) return finalize_rows(ctx, res);
  PhaseClock pc;
  FinalizeDesc& fd = res->fd;
  cudaStream_t s = ctx->stream;
  // Upper bound of result rows: every slot could be occupied; count first to size the output.
  // (k_finalize with max_out == 0 only counts.)
  DevBuf& cnt = res->cnt;
  unsigned int n_groups = res->n_groups;
  if (!res->groups_known) {
    CUDA_TRY(cnt.alloc(16, ctx->stream));
    CUDA_TRY(cudaMemsetAsync(cnt.p, 0, 16, s));
    res->cnt_ptr = static_cast<unsigned int*>(cnt.p);
    CUDA_TRY(launch_count_groups(fd, res->cnt_ptr, s));
    CUDA_TRY(cudaMemcpyAsync(&n_groups, cnt.p, 4, cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaStreamSynchronize(s));
    res->stats.kernel_launches += 1;
  }
  res->stats.groups = n_groups;
  const size_t G = n_groups;
  const int nk = fd.n_keys, na = fd.n_aggs;
  // every result column lands in its own page-locked block of the context's pool; int64 keys and aggregates hand
  // that block to the Arrow consumer as it is (returned to the pool on release), dictionary keys are re-indexed
  std::vector<PinnedBlock> blocks(size_t(nk + na));
  if (G > 0) {
    DevBuf out;
    size_t bytes = (size_t(nk) + size_t(na) + 1) * G * 8;
    CUDA_TRY(out.alloc(bytes, ctx->stream));
    CUDA_TRY(cudaMemsetAsync(res->cnt_ptr, 0, 16, s));
    fd.out_count = res->cnt_ptr;
    fd.max_out = n_groups;
    fd.out_keys = static_cast<long long*>(out.p);
    fd.out_aggs = fd.out_keys + size_t(nk) * G;
    fd.out_rows = reinterpret_cast<unsigned long long*>(fd.out_aggs + size_t(na) * G);
    CUDA_TRY(launch_finalize(fd, s));
    res->stats.kernel_launches += 1;
    for (int c = 0; c < nk + na; c++) {
      blocks[size_t(c)] = PinnedBlock(ctx->pinned, G * 8);
      if (!blocks[size_t(c)]) return fail(FGPU_ERR_OOM, "page-locked memory for the result columns");
      CUDA_TRY(cudaMemcpyAsync(blocks[size_t(c)].get(), fd.out_keys + size_t(c) * G, G * 8, cudaMemcpyDeviceToHost, s));
    }
    CUDA_TRY(cudaStreamSynchronize(s));
    res->stats.d2h_bytes += (size_t(nk) + size_t(na)) * G * 8;
  }
  CUDA_TRY(cudaEventRecord(ctx->ev[3], s));
  CUDA_TRY(cudaEventSynchronize(ctx->ev[3]));
  float ms = 0;
  cudaEventElapsedTime(&ms, ctx->ev[0], ctx->ev[3]);
  res->stats.total_device_ms = ms;
  pc.mark("finalize_device");

  // ---- build Arrow columns (aggregate.go:551-625: group columns first, then aggregates) --------
  std::vector<OwnedColumn> cols;
  for (int c = 0, o = 0; c < nk + na; c++) {
    const bool key = c < nk;
    const uint8_t unique = key ? UC_NONE : res->qd.aggs[c - nk].unique;
    if (unique == UC_HI) continue;  // the validity of the Unique before it
    OwnedColumn col;
    col.name = key ? res->shape.keys[size_t(c)].name : res->shape.agg_names[size_t(o)];
    col.length = int64_t(G);
    if (key && res->shape.keys[size_t(c)].is_bool) {  // codes (1 false, 2 true) packed into bits in place
      bool_key_column(col, reinterpret_cast<long long*>(blocks[size_t(c)].get()), G);
      if (G) {
        col.ext = blocks[size_t(c)].get();
        col.ext_keep = std::move(blocks[size_t(c)]).keep();
      }
    } else if (key && !res->shape.keys[size_t(c)].is_int64) {  // codes (id + 1, 0 = NULL) re-indexed into col.data
      dict_key_column(col, reinterpret_cast<const long long*>(blocks[size_t(c)].get()), G, nullptr, res->shape.keys[size_t(c)].dict_snapshot,
                      KeyDict::kUsed);
    } else {
      col.format = !key && res->shape.agg_is_float[size_t(o)] ? "g" : "l";
      if (unique == UC_LO) validity_from_bytes(col, blocks[size_t(c + 1)].get(), G);
      if (G) {
        col.ext = blocks[size_t(c)].get();
        col.ext_keep = std::move(blocks[size_t(c)]).keep();
      }
    }
    o += key ? 0 : 1;
    cols.push_back(std::move(col));
  }
  res->stats.algorithmic_bytes += (size_t(nk) + size_t(na)) * G * 8;
  res->finish(std::move(cols), G);
  res->table.reset();
  res->aux.reset();
  res->cnt.reset();
  pc.mark("arrow");
  pc.flush("finalize");
  return FGPU_OK;
}

// One partial table to fold: a table of the result's layout at `slots` slots.
struct Partial {
  const void* table;
  uint32_t slots;
};

// Folds partial tables into a fresh table of `slots` slots (k_table_init, then one k_merge per partial) and installs it
// in the result: table, table_bytes, qd, fd.  zero_counters: whether the table init zeroes the query's counters.
int32_t fold_partials(fgpu_ctx* ctx, fgpu_result* res, uint32_t slots, const std::vector<Partial>& parts, bool zero_counters) {
  cudaStream_t s = ctx->stream;
  QueryDesc qd = res->qd;
  qd.table_slots = slots;
  size_t off_aggs, off_tags, off_keys;
  const size_t tbytes = table_layout(qd, &off_aggs, &off_tags, &off_keys);
  DevBuf merged;
  CUDA_TRY(merged.alloc(tbytes + 128, s));  // (slack for the 16-byte exchange copies)
  bind_table(&qd, static_cast<uint8_t*>(merged.p));
  CUDA_TRY(launch_table_init(qd, s, zero_counters));
  for (const Partial& p : parts) CUDA_TRY(launch_merge(qd, p.table, p.slots, s));
  std::swap(res->table.p, merged.p);
  std::swap(res->table.n, merged.n);
  res->table_bytes = tbytes;
  res->qd = qd;
  res->fd.table_slots = slots;
  bind_finalize(&res->fd, qd);
  return FGPU_OK;
}

// Behind a merge: counts the final table's groups (when the result counts them on the device), reads the counters back
// into the context's scratch (to *counters when asked) and fails on a hash table overflow.
int32_t count_merged(fgpu_ctx* ctx, fgpu_result* res, const unsigned long long** counters) {
  cudaStream_t s = ctx->stream;
  if (res->cnt_ptr) {
    CUDA_TRY(cudaMemsetAsync(res->cnt_ptr, 0, 16, s));
    CUDA_TRY(launch_count_groups(res->fd, res->cnt_ptr, s));
    res->stats.kernel_launches++;
  }
  CUDA_TRY(ctx->ensure_scratch(128));
  unsigned long long* c = reinterpret_cast<unsigned long long*>(ctx->scratch);
  CUDA_TRY(cudaMemcpyAsync(c, res->qd.counters, 64 + 16, cudaMemcpyDeviceToHost, s));
  CUDA_TRY(cudaStreamSynchronize(s));
  if (c[1]) return fail(FGPU_ERR_UNSUPPORTED, "aggregate hash table overflow while merging partials");
  if (res->cnt_ptr) {
    res->n_groups = static_cast<unsigned int>(c[8] & 0xffffffffull);
    res->groups_known = true;
  }
  if (counters) *counters = c;
  return FGPU_OK;
}

// Second half of a collective Execute: wait for the peers, merge, bring the final result to the host.
int32_t collective_end(fgpu_ctx* ctx, fgpu_result* res) {
  if (!res->pending) return fail(FGPU_ERR_INVALID, "no collective Execute pending on this result");
  res->pending = false;
  if (ExecCache* x = static_cast<ExecCache*>(res->pending_cached)) {
    if (int32_t rc = cached_merge_tail(ctx, *x, res->pending_seq, res->pending_bytes)) return rc;
    CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    const unsigned long long* counters = reinterpret_cast<const unsigned long long*>(x->pinned.get() + 32);
    res->stats.d2h_bytes += x->out_bytes;
    if (int32_t rcc = comm_check(counters[3])) return rcc;
    return finalize_dense_host(res, *x);
  }
  const QueryDesc& qd = res->qd;
  int32_t rc = comm_wait_merge(ctx, qd, res->table.p, res->pending_seq, res->pending_bytes);
  if (rc) return rc;
  if (qd.table_mode != TM_DENSE) {  // hash tables: fold every rank's slot, at its own size, into a fresh table
    uint32_t src_slots[kMaxRanks];
    if (int32_t rcs = hash_partial_slots(ctx, qd, res->pending_seq, src_slots)) return rcs;
    uint64_t total = 0;
    std::vector<Partial> parts;
    for (int r = 0; r < ctx->comm.n; r++) {
      total += src_slots[r];
      parts.push_back({ctx->comm.mailbox + ctx->comm.data_off(res->pending_seq & 1u, r), src_slots[r]});
    }
    // (counters[3] carries the exchange's error: the init leaves the counters alone)
    if (int32_t rcf = fold_partials(ctx, res, hash_slots(total), parts, /*zero_counters=*/false)) return rcf;
  }
  const unsigned long long* counters = nullptr;
  if (int32_t rcc = count_merged(ctx, res, &counters)) return rcc;
  if (int32_t rcc = comm_check(counters[3])) return rcc;
  return finalize_result(ctx, res);
}

}  // namespace

// =====================================================================================================
// extern "C"
// =====================================================================================================
// No C++ exception crosses the C ABI: every entry point that returns a status runs inside this guard.
#define API_TRY try {
#define API_CATCH                                                                      \
  }                                                                                    \
  catch (const std::bad_alloc&) { return fail(FGPU_ERR_OOM, "out of host memory"); }   \
  catch (const std::exception& ex) { return fail(FGPU_ERR_INVALID, std::string("internal error: ") + ex.what()); } \
  catch (...) { return fail(FGPU_ERR_INVALID, "internal error"); }

extern "C" {

const char* fgpu_last_error(void) { return g_err.c_str(); }
int32_t fgpu_abi_version(void) { return FGPU_ABI_VERSION; }

int32_t fgpu_init(const fgpu_config* cfg, fgpu_ctx** out) {
  API_TRY
  if (!cfg || !out) return fail(FGPU_ERR_INVALID, "null argument");
  if (cfg->abi_version != FGPU_ABI_VERSION) return fail(FGPU_ERR_INVALID, "ABI version mismatch");
  if (cfg->tile_rows != 0 && cfg->tile_rows != kTileRows) return fail(FGPU_ERR_INVALID, "tile_rows must be 0 (default)");
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n == 0) {
    cudaGetLastError();
    return fail(FGPU_ERR_NO_DEVICE, std::string("no CUDA device: ") + (e != cudaSuccess ? cudaGetErrorString(e) : "device count is 0"));
  }
  if (cfg->device < 0 || cfg->device >= n) return fail(FGPU_ERR_INVALID, "device ordinal out of range");
  CUDA_TRY(cudaSetDevice(cfg->device));
  auto ctx = std::make_unique<fgpu_ctx>();
  ctx->device = cfg->device;
  cudaDeviceProp prop;
  CUDA_TRY(cudaGetDeviceProperties(&prop, cfg->device));
  ctx->sm_count = prop.multiProcessorCount;
  CUDA_TRY(cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking));
  {
    cudaMemPool_t pool;
    CUDA_TRY(cudaDeviceGetDefaultMemPool(&pool, cfg->device));
    uint64_t keep = ~0ull;  // freed blocks stay in the pool: allocation is a pointer bump afterwards
    CUDA_TRY(cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep));
  }
  for (auto& ev : ctx->ev) CUDA_TRY(cudaEventCreate(&ev));
  *out = ctx.release();
  return FGPU_OK;
  API_CATCH
}

int32_t fgpu_shutdown(fgpu_ctx* ctx) {
  API_TRY
  if (!ctx) return FGPU_OK;
  cudaSetDevice(ctx->device);
  if (ctx->comm.mailbox) {
    for (int r = 0; r < ctx->comm.n; r++)
      if (ctx->comm.peer_ipc[r] && ctx->comm.peer[r]) cudaIpcCloseMemHandle(ctx->comm.peer[r]);
    cudaFree(ctx->comm.mailbox);
    ctx->comm = Comm{};
  }
  for (auto& kv : ctx->plans) kv.second->plan_cache.reset();  // device state of compiled plans (queries still held by the caller stay valid handles)
  ctx->plans.clear();
  for (auto& t : ctx->tables)
    for (auto& p : t.second.parts) free_part(ctx, p.get());
  if (ctx->stream) cudaStreamSynchronize(ctx->stream);
  for (auto& ev : ctx->ev)
    if (ev) cudaEventDestroy(ev);
  if (ctx->stream) cudaStreamDestroy(ctx->stream);
  if (ctx->scratch) cudaFreeHost(ctx->scratch);
  if (ctx->arena) cudaFreeHost(ctx->arena);
  delete ctx;
  return FGPU_OK;
  API_CATCH
}

int32_t fgpu_part_put_parquet(fgpu_ctx* ctx, const char* table, uint64_t part_id, uint64_t tx, const uint8_t* file,
                              uint64_t len, int32_t flags) {
  API_TRY
  if (!ctx || !table || !file) return fail(FGPU_ERR_INVALID, "null argument");
  if (flags != FGPU_PUT_DEFAULT && flags != FGPU_PUT_BORROW_PINNED) return fail(FGPU_ERR_INVALID, "unknown put flags");
  std::lock_guard<std::mutex> lk(ctx->mu);
  PhaseClock pc;
  struct PutTail { PhaseClock& pc; ~PutTail() { pc.mark("put"); pc.flush("put"); } } put_tail{pc};
  CUDA_TRY(cudaSetDevice(ctx->device));
  Table& t = ctx->tables[table];
  for (auto& p : t.parts)
    if (p->id == part_id) return fail(FGPU_ERR_INVALID, "part id already registered");
  auto part = std::make_unique<Part>();
  part->id = part_id;
  part->tx = tx;
  part->borrowed = flags == FGPU_PUT_BORROW_PINNED;
  std::string err;
  if (!open_part(file, len, part.get(), &err)) return fail(FGPU_ERR_PARQUET, err);
  if (!part->borrowed) {
    // The caller may reuse the buffer on return: every column goes to the device now (host images built in
    // parallel, one worker per column; PLAIN string pages interned in one batch).
    if (int32_t rc = upload_part(ctx, &t, part.get())) return rc;
    part->file = nullptr;
  }
  t.parts.push_back(std::move(part));
  t.epoch = ++ctx->epoch_counter;
  return FGPU_OK;
  API_CATCH
}

int32_t fgpu_part_put_arrow(fgpu_ctx* ctx, const char* table, uint64_t part_id, uint64_t tx, struct ArrowSchema* schema,
                            struct ArrowArray* array) {
  API_TRY
  // the library owns both structs from here on, whatever happens
  struct Release {
    ArrowSchema* s; ArrowArray* a;
    ~Release() {
      if (s && s->release) s->release(s);
      if (a && a->release) a->release(a);
    }
  } rel{schema, array};
  if (!ctx || !table || !schema || !array) return fail(FGPU_ERR_INVALID, "null argument");
  std::lock_guard<std::mutex> lk(ctx->mu);
  CUDA_TRY(cudaSetDevice(ctx->device));
  Table& t = ctx->tables[table];
  for (auto& p : t.parts)
    if (p->id == part_id) return fail(FGPU_ERR_INVALID, "part id already registered");
  auto part = std::make_unique<Part>();
  part->id = part_id;
  part->tx = tx;
  std::string err;
  part->arrow = true;
  if (!build_arrow_part(&t, part.get(), schema, array, &err)) return fail(FGPU_ERR_UNSUPPORTED, "Arrow part: " + err);
  // the record's buffers go away on return: every column image is uploaded now
  if (int32_t rc = upload_part(ctx, &t, part.get())) return rc;
  t.parts.push_back(std::move(part));
  t.epoch = ++ctx->epoch_counter;
  return FGPU_OK;
  API_CATCH
}

int32_t fgpu_part_drop(fgpu_ctx* ctx, const char* table, uint64_t part_id) {
  API_TRY
  if (!ctx || !table) return fail(FGPU_ERR_INVALID, "null argument");
  std::lock_guard<std::mutex> lk(ctx->mu);
  auto it = ctx->tables.find(table);
  if (it == ctx->tables.end()) return fail(FGPU_ERR_NOT_FOUND, std::string("table not found: ") + table);
  auto& parts = it->second.parts;
  for (size_t i = 0; i < parts.size(); i++) {
    if (parts[i]->id == part_id) {
      cudaSetDevice(ctx->device);
      cudaStreamSynchronize(ctx->stream);
      release_staging(ctx);
      free_part(ctx, parts[i].get());
      parts.erase(parts.begin() + long(i));
      it->second.epoch = ++ctx->epoch_counter;
      return FGPU_OK;
    }
  }
  return fail(FGPU_ERR_NOT_FOUND, "part not found");
  API_CATCH
}

int32_t fgpu_table_drop(fgpu_ctx* ctx, const char* table) {
  API_TRY
  if (!ctx || !table) return fail(FGPU_ERR_INVALID, "null argument");
  std::lock_guard<std::mutex> lk(ctx->mu);
  auto it = ctx->tables.find(table);
  if (it == ctx->tables.end()) return FGPU_OK;
  PhaseClock pc;
  cudaSetDevice(ctx->device);
  cudaStreamSynchronize(ctx->stream);
  release_staging(ctx);
  for (auto& p : it->second.parts) free_part(ctx, p.get());
  ctx->tables.erase(it);
  pc.mark("drop");
  pc.flush("drop");
  return FGPU_OK;
  API_CATCH
}

int32_t fgpu_query_prepare(fgpu_ctx* ctx, const fgpu_plan* plan, fgpu_query** out) {
  API_TRY
  if (!ctx || !plan || !out || !plan->table) return fail(FGPU_ERR_INVALID, "null argument");
  if (plan->kind != FGPU_PLAN_AGGREGATE && plan->kind != FGPU_PLAN_DISTINCT && plan->kind != FGPU_PLAN_FILTER)
    return fail(FGPU_ERR_INVALID, "unknown plan kind");
  auto q = std::make_shared<QueryPlan>();
  q->ctx = ctx;
  q->table = plan->table;
  q->kind = plan->kind;
  q->filter = plan->filter;
  // the plan's text: two prepared queries with the same signature share one QueryPlan (and its compiled state)
  std::string sig;
  auto put = [&](const void* p, size_t n) { sig.append(static_cast<const char*>(p), n); };
  auto put_str = [&](const std::string& v) { const uint64_t n = v.size(); put(&n, 8); sig += v; };
  put_str(q->table);
  put(&plan->kind, 4);
  put(&plan->filter, 4);
  auto check = [&](int32_t i) { return i >= 0 && i < plan->n_exprs; };
  for (int32_t i = 0; i < plan->n_exprs; i++) {
    const fgpu_expr& e = plan->exprs[i];
    ExprNode n;
    n.kind = e.kind;
    n.op = e.op;
    n.left = e.left;
    n.right = e.right;
    put(&e.kind, 4); put(&e.op, 4); put(&e.left, 4); put(&e.right, 4);
    if (e.kind == FGPU_EXPR_COLUMN || e.kind == FGPU_EXPR_DYNCOLUMN) {
      if (!e.name) return fail(FGPU_ERR_INVALID, "column expression without a name");
      n.name = e.name;
      put_str(n.name);
    } else if (e.kind == FGPU_EXPR_LITERAL) {
      n.lit_type = e.literal.type;
      n.lit_i = e.literal.i64;
      n.lit_f = e.literal.f64;
      if (e.literal.type == FGPU_SCALAR_STRING) {
        if (e.literal.len && !e.literal.bytes) return fail(FGPU_ERR_INVALID, "string literal without bytes");
        n.lit_bytes.assign(reinterpret_cast<const char*>(e.literal.bytes), size_t(e.literal.len));
      }
      put(&n.lit_type, 4); put(&n.lit_i, 8); put(&n.lit_f, 8);
      put_str(n.lit_bytes);
    } else if (e.kind == FGPU_EXPR_BINARY) {
      if (!check(e.left) || !check(e.right) || e.left >= i || e.right >= i)
        return fail(FGPU_ERR_INVALID, "binary expression children must precede their parent");
      n.match = e.match;
      n.match_user = e.match_user;
      const void* fn = reinterpret_cast<const void*>(e.match);
      put(&fn, sizeof fn); put(&e.match_user, sizeof e.match_user);  // a different matcher is a different plan
    } else {
      return fail(FGPU_ERR_INVALID, "unknown expression kind");
    }
    q->exprs.push_back(std::move(n));
  }
  if (plan->filter >= 0 && !check(plan->filter)) return fail(FGPU_ERR_INVALID, "filter index out of range");
  for (int32_t i = 0; i < plan->n_group_by; i++) {
    if (!check(plan->group_by[i])) return fail(FGPU_ERR_INVALID, "group-by index out of range");
    q->group_by.push_back(plan->group_by[i]);
    put(&plan->group_by[i], 4);
  }
  if (plan->kind != FGPU_PLAN_AGGREGATE && plan->n_aggs != 0) return fail(FGPU_ERR_INVALID, "DISTINCT / FILTER plan with aggregates");
  if (plan->kind == FGPU_PLAN_AGGREGATE && plan->n_aggs == 0) return fail(FGPU_ERR_INVALID, "AGGREGATE plan without aggregates");
  sig += "|";
  for (int32_t i = 0; i < plan->n_aggs; i++) {
    if (!check(plan->aggs[i].expr)) return fail(FGPU_ERR_INVALID, "aggregate expression index out of range");
    q->aggs.push_back(plan->aggs[i]);
    put(&plan->aggs[i].func, 4); put(&plan->aggs[i].expr, 4);
  }
  auto handle = std::make_unique<fgpu_query>();
  handle->ctx = ctx;
  {
    std::lock_guard<std::mutex> lk(ctx->mu);
    auto it = ctx->plans.find(sig);
    if (it != ctx->plans.end()) {
      handle->plan = it->second;
    } else {
      if (ctx->plans.size() >= 256) {  // bounded: forget the plans nobody holds any more, then everything
        CUDA_TRY(cudaSetDevice(ctx->device));
        for (auto p = ctx->plans.begin(); p != ctx->plans.end();) p = p->second.use_count() == 1 ? ctx->plans.erase(p) : std::next(p);
        if (ctx->plans.size() >= 256) ctx->plans.clear();
      }
      ctx->plans.emplace(std::move(sig), q);
      handle->plan = std::move(q);
    }
  }
  *out = handle.release();
  return FGPU_OK;
  API_CATCH
}

int32_t fgpu_query_free(fgpu_query* q) {
  API_TRY
  if (q && q->ctx) {  // the last reference to a plan may own device state
    std::lock_guard<std::mutex> lk(q->ctx->mu);
    cudaSetDevice(q->ctx->device);
    q->plan.reset();
  }
  delete q;
  return FGPU_OK;
  API_CATCH
}

int32_t fgpu_query_execute(fgpu_ctx* ctx, fgpu_query* q, uint64_t tx_watermark, fgpu_result** out) {
  API_TRY
  if (!ctx || !q || !out) return fail(FGPU_ERR_INVALID, "null argument");
  std::lock_guard<std::mutex> lk(ctx->mu);
  CUDA_TRY(cudaSetDevice(ctx->device));
  auto res = std::make_unique<fgpu_result>();
  res->ctx = ctx;
  int32_t rc = run_scan(ctx, *q->plan, tx_watermark, res.get(), /*count_groups=*/true, /*cacheable=*/true);
  if (rc) return rc;
  if (!res->finalized) rc = finalize_result(ctx, res.get());
  if (rc) return rc;
  *out = res.release();
  return FGPU_OK;
  API_CATCH
}

int32_t fgpu_query_execute_partial(fgpu_ctx* ctx, fgpu_query* q, uint64_t tx_watermark, fgpu_result** out, void** dev_ptr,
                                   uint64_t* nbytes) {
  API_TRY
  if (!ctx || !q || !out || !dev_ptr || !nbytes) return fail(FGPU_ERR_INVALID, "null argument");
  std::lock_guard<std::mutex> lk(ctx->mu);
  CUDA_TRY(cudaSetDevice(ctx->device));
  auto res = std::make_unique<fgpu_result>();
  res->ctx = ctx;
  if (q->plan->kind == FGPU_PLAN_FILTER) return fail(FGPU_ERR_INVALID, "rows plans have no partial table: execute them per rank");
  int32_t rc = run_scan(ctx, *q->plan, tx_watermark, res.get());
  if (rc) return rc;
  *dev_ptr = res->table.p;
  *nbytes = res->table_bytes;
  *out = res.release();
  return FGPU_OK;
  API_CATCH
}

int32_t fgpu_result_merge_partials(fgpu_ctx* ctx, fgpu_result* r, const void* gathered, uint64_t nbytes, int32_t n) {
  API_TRY
  if (!ctx || !r) return fail(FGPU_ERR_INVALID, "null argument");
  if (r->finalized) return fail(FGPU_ERR_INVALID, "result already finalised");
  std::lock_guard<std::mutex> lk(ctx->mu);
  CUDA_TRY(cudaSetDevice(ctx->device));
  if (n > 0) {
    if (!gathered) return fail(FGPU_ERR_INVALID, "null gathered buffer");
    if (nbytes != r->table_bytes) return fail(FGPU_ERR_INVALID, "partial table size differs between ranks (dictionaries not preloaded identically?)");
    // Start from an empty table and fold every rank's partial in, this rank's own included.  A hash table takes the
    // groups of n partials: it is sized for n times this rank's slots.
    const uint32_t src_slots = r->qd.table_slots;
    std::vector<Partial> parts;
    for (int32_t i = 0; i < n; i++) parts.push_back({static_cast<const uint8_t*>(gathered) + size_t(i) * nbytes, src_slots});
    const uint32_t slots = r->qd.table_mode == TM_DENSE ? src_slots : hash_slots(uint64_t(n) * src_slots);
    if (int32_t rc = fold_partials(ctx, r, slots, parts, /*zero_counters=*/true)) return rc;
    r->stats.kernel_launches += uint32_t(n);  // k_merge
    // the groups are counted right behind the merges, so that finalisation needs one host round trip less
    if (int32_t rc = count_merged(ctx, r, nullptr)) return rc;
  }
  return finalize_result(ctx, r);
  API_CATCH
}

int32_t fgpu_comm_export(fgpu_ctx* ctx, int32_t rank, int32_t n_ranks, uint64_t slot_bytes, uint8_t* handle) {
  API_TRY
  if (!ctx || !handle) return fail(FGPU_ERR_INVALID, "null argument");
  if (n_ranks < 1 || n_ranks > kMaxRanks || rank < 0 || rank >= n_ranks) return fail(FGPU_ERR_INVALID, "rank / n_ranks out of range");
  std::lock_guard<std::mutex> lk(ctx->mu);
  CUDA_TRY(cudaSetDevice(ctx->device));
  Comm& cm = ctx->comm;
  if (cm.mailbox) return fail(FGPU_ERR_INVALID, "communicator already exported: fgpu_comm_close first");
  cm.rank = rank;
  cm.n = n_ranks;
  cm.slot_bytes = (std::max<uint64_t>(slot_bytes, 4096) + 255) & ~uint64_t(255);
  cm.total = kCommDataOff + 2 * uint64_t(n_ranks) * cm.slot_bytes;
  cm.seq = 0;
  void* p = nullptr;
  CUDA_TRY(cudaMalloc(&p, cm.total));  // (cudaMalloc, not the stream-ordered pool: the allocation is exported through CUDA IPC)
  cm.mailbox = static_cast<uint8_t*>(p);
  CUDA_TRY(cudaMemset(cm.mailbox, 0, kCommDataOff));
  CommHandle h{};
  h.magic = kCommMagic;
  h.device = ctx->device;
  h.pid = uint64_t(getpid());
  h.ptr = uint64_t(reinterpret_cast<uintptr_t>(cm.mailbox));
  h.total = cm.total;
  h.slot_bytes = cm.slot_bytes;
  h.n = n_ranks;
  h.rank = rank;
  CUDA_TRY(cudaIpcGetMemHandle(&h.ipc, cm.mailbox));
  std::memset(handle, 0, FGPU_COMM_HANDLE_BYTES);
  std::memcpy(handle, &h, sizeof h);
  return FGPU_OK;
  API_CATCH
}

int32_t fgpu_comm_open(fgpu_ctx* ctx, const uint8_t* all_handles) {
  API_TRY
  if (!ctx || !all_handles) return fail(FGPU_ERR_INVALID, "null argument");
  std::lock_guard<std::mutex> lk(ctx->mu);
  CUDA_TRY(cudaSetDevice(ctx->device));
  Comm& cm = ctx->comm;
  if (!cm.mailbox) return fail(FGPU_ERR_INVALID, "fgpu_comm_export first");
  if (cm.open) return fail(FGPU_ERR_INVALID, "communicator already open");
  for (int r = 0; r < cm.n; r++) {
    CommHandle h;
    std::memcpy(&h, all_handles + size_t(r) * FGPU_COMM_HANDLE_BYTES, sizeof h);
    if (h.magic != kCommMagic || h.rank != r || h.n != cm.n || h.slot_bytes != cm.slot_bytes)
      return fail(FGPU_ERR_INVALID, "handle " + std::to_string(r) + " does not belong to this communicator (rank order, n_ranks and slot_bytes must agree)");
    if (r == cm.rank) {
      cm.peer[r] = cm.mailbox;
      cm.peer_ipc[r] = false;
    } else if (h.pid == uint64_t(getpid())) {  // another context of this process: plain peer access
      if (h.device != ctx->device) {
        cudaError_t e = cudaDeviceEnablePeerAccess(h.device, 0);
        if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) {
          cudaGetLastError();
          return fail(FGPU_ERR_CUDA, std::string("peer access to device ") + std::to_string(h.device) + ": " + cudaGetErrorString(e));
        }
        cudaGetLastError();
      }
      cm.peer[r] = reinterpret_cast<uint8_t*>(uintptr_t(h.ptr));
      cm.peer_ipc[r] = false;
    } else {
      void* p = nullptr;
      CUDA_TRY(cudaIpcOpenMemHandle(&p, h.ipc, cudaIpcMemLazyEnablePeerAccess));
      cm.peer[r] = static_cast<uint8_t*>(p);
      cm.peer_ipc[r] = true;
    }
  }
  cm.open = true;
  return FGPU_OK;
  API_CATCH
}

int32_t fgpu_comm_close(fgpu_ctx* ctx) {
  API_TRY
  if (!ctx) return FGPU_OK;
  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaSetDevice(ctx->device);
  Comm& cm = ctx->comm;
  if (ctx->stream) cudaStreamSynchronize(ctx->stream);
  for (int r = 0; r < cm.n; r++)
    if (cm.peer_ipc[r] && cm.peer[r]) cudaIpcCloseMemHandle(cm.peer[r]);
  if (cm.mailbox) cudaFree(cm.mailbox);
  cudaGetLastError();
  cm = Comm{};
  return FGPU_OK;
  API_CATCH
}

int32_t fgpu_query_execute_collective(fgpu_ctx* ctx, fgpu_query* q, uint64_t tx_watermark, fgpu_result** out) {
  API_TRY
  if (!ctx || !q || !out) return fail(FGPU_ERR_INVALID, "null argument");
  std::lock_guard<std::mutex> lk(ctx->mu);
  CUDA_TRY(cudaSetDevice(ctx->device));
  auto res = std::make_unique<fgpu_result>();
  res->ctx = ctx;
  // a cached plan: scan -> push -> wait -> merge -> one copy back, one synchronisation; the first run of a plan
  // pushes, synchronises once more for its own bookkeeping and then runs the merge half
  int32_t rc = run_scan(ctx, *q->plan, tx_watermark, res.get(), /*count_groups=*/false, /*cacheable=*/true, /*collective=*/1);
  if (rc) return rc;
  if (res->pending) rc = collective_end(ctx, res.get());
  if (rc) return rc;
  *out = res.release();
  return FGPU_OK;
  API_CATCH
}

int32_t fgpu_query_execute_collective_begin(fgpu_ctx* ctx, fgpu_query* q, uint64_t tx_watermark, fgpu_result** out) {
  API_TRY
  if (!ctx || !q || !out) return fail(FGPU_ERR_INVALID, "null argument");
  std::lock_guard<std::mutex> lk(ctx->mu);
  CUDA_TRY(cudaSetDevice(ctx->device));
  auto res = std::make_unique<fgpu_result>();
  res->ctx = ctx;
  int32_t rc = run_scan(ctx, *q->plan, tx_watermark, res.get(), /*count_groups=*/false, /*cacheable=*/true, /*collective=*/2);
  if (rc) return rc;
  res->plan_keep = q->plan->plan_cache;
  *out = res.release();
  return FGPU_OK;
  API_CATCH
}

int32_t fgpu_query_execute_collective_end(fgpu_ctx* ctx, fgpu_result* r) {
  API_TRY
  if (!ctx || !r) return fail(FGPU_ERR_INVALID, "null argument");
  std::lock_guard<std::mutex> lk(ctx->mu);
  CUDA_TRY(cudaSetDevice(ctx->device));
  return collective_end(ctx, r);
  API_CATCH
}

int32_t fgpu_result_partial_is_additive(const fgpu_result* r, int32_t* out) {
  API_TRY
  if (!r || !out) return fail(FGPU_ERR_INVALID, "null argument");
  bool add = !r->rows_plan && r->qd.table_mode == TM_DENSE;
  for (int a = 0; a < r->qd.n_aggs && add; a++)
    if (r->qd.aggs[a].func != FGPU_AGG_COUNT && !(r->qd.aggs[a].func == FGPU_AGG_SUM && !r->qd.aggs[a].is_float)) add = false;
  *out = add ? 1 : 0;
  return FGPU_OK;
  API_CATCH
}

int32_t fgpu_rowgroup_leaf_mode(int32_t op, int64_t literal, int32_t has_bounds, int64_t min_value, int64_t max_value, int64_t null_count,
                                int64_t num_values, int32_t* out_mode) {
  API_TRY
  if (!out_mode) return fail(FGPU_ERR_INVALID, "null argument");
  if (op < FGPU_OP_EQ || op > FGPU_OP_GT_EQ) return fail(FGPU_ERR_INVALID, "not a comparison operator");
  int64_t lo, hi;
  bool neg;
  canonical_int_range(op, literal, &lo, &hi, &neg);
  *out_mode = chunk_leaf_mode(lo, hi, neg, has_bounds != 0, min_value, max_value, null_count, num_values);
  return FGPU_OK;
  API_CATCH
}

int32_t fgpu_xxhash64(const uint8_t* data, uint64_t len, uint64_t seed, uint64_t* out) {
  API_TRY
  if ((!data && len) || !out) return fail(FGPU_ERR_INVALID, "null argument");
  *out = xxhash64(data, size_t(len), seed);
  return FGPU_OK;
  API_CATCH
}

int32_t fgpu_lz4_raw_inflate(const uint8_t* src, uint64_t len, uint8_t* dst, uint64_t cap, uint64_t* out_len) {
  API_TRY
  if ((!src && len) || !out_len) return fail(FGPU_ERR_INVALID, "null argument");
  *out_len = 0;
  std::string err;
  if (!parse_lz4_raw(src, len, cap, &err)) return fail(FGPU_ERR_PARQUET, err);
  if (dst) {
    unpack_lz4_raw(src, len, dst, cap);
    *out_len = cap;
  }
  return FGPU_OK;
  API_CATCH
}

int32_t fgpu_bloom_check(const uint8_t* bitset, uint64_t nbytes, uint64_t hash, int32_t* out_may_contain) {
  API_TRY
  if (!bitset || !out_may_contain) return fail(FGPU_ERR_INVALID, "null argument");
  if (nbytes < 32 || nbytes % 32 != 0 || nbytes > 0xffffffffull) return fail(FGPU_ERR_INVALID, "a split-block filter is a multiple of 32 bytes");
  *out_may_contain = sbbf_check(bitset, uint32_t(nbytes), hash) ? 1 : 0;
  return FGPU_OK;
  API_CATCH
}

int32_t fgpu_bloom_insert(uint8_t* bitset, uint64_t nbytes, uint64_t hash) {
  API_TRY
  if (!bitset) return fail(FGPU_ERR_INVALID, "null argument");
  if (nbytes < 32 || nbytes % 32 != 0 || nbytes > 0xffffffffull) return fail(FGPU_ERR_INVALID, "a split-block filter is a multiple of 32 bytes");
  sbbf_insert(bitset, uint32_t(nbytes), hash);
  return FGPU_OK;
  API_CATCH
}

int32_t fgpu_parquet_rowgroup_may_match_eq(const uint8_t* file, uint64_t len, int32_t row_group, const char* column, int32_t lit_type,
                                           int64_t lit_i64, double lit_f64, const uint8_t* lit_bytes, uint64_t lit_len, int32_t* out) {
  API_TRY
  if (!file || !column || !out) return fail(FGPU_ERR_INVALID, "null argument");
  Part part;
  std::string err;
  if (!open_part(file, len, &part, &err)) return fail(FGPU_ERR_PARQUET, err);
  if (row_group < 0 || size_t(row_group) >= part.rgs.size()) return fail(FGPU_ERR_INVALID, "no such row group");
  QueryPlan q;
  ExprNode col, lit, eq;
  col.kind = FGPU_EXPR_COLUMN;
  col.name = column;
  lit.kind = FGPU_EXPR_LITERAL;
  lit.lit_type = lit_type;
  lit.lit_i = lit_i64;
  lit.lit_f = lit_f64;
  if (lit_bytes && lit_len) lit.lit_bytes.assign(reinterpret_cast<const char*>(lit_bytes), size_t(lit_len));
  eq.kind = FGPU_EXPR_BINARY;
  eq.op = FGPU_OP_EQ;
  eq.left = 0;
  eq.right = 1;
  q.exprs = {col, lit, eq};
  *out = rg_may_match(q, 2, part.rgs[size_t(row_group)]) ? 1 : 0;
  return FGPU_OK;
  API_CATCH
}

int32_t fgpu_result_next(fgpu_result* r, struct ArrowSchema* out_schema, struct ArrowArray* out_array) {
  API_TRY
  if (!r || !out_schema || !out_array) return fail(FGPU_ERR_INVALID, "null argument");
  if (!r->finalized) return fail(FGPU_ERR_INVALID, r->pending ? "collective Execute pending: call fgpu_query_execute_collective_end first"
                                                               : "partial result: call fgpu_result_merge_partials first");
  if (r->next >= r->records.size()) return fail(FGPU_ERR_END, "no more records");
  export_record(std::move(r->records[r->next]), r->record_rows[r->next], out_schema, out_array);
  r->next++;
  return FGPU_OK;
  API_CATCH
}

int32_t fgpu_result_stats(const fgpu_result* r, fgpu_stats* out) {
  API_TRY
  if (!r || !out) return fail(FGPU_ERR_INVALID, "null argument");
  *out = r->stats;
  return FGPU_OK;
  API_CATCH
}

int32_t fgpu_result_free(fgpu_result* r) {
  API_TRY
  if (r) {
    if (r->ctx) cudaSetDevice(r->ctx->device);
    delete r;
  }
  return FGPU_OK;
  API_CATCH
}

int32_t fgpu_host_alloc(uint64_t bytes, void** out) {
  API_TRY
  if (!out) return fail(FGPU_ERR_INVALID, "null argument");
  void* p = nullptr;
  cudaError_t e = cudaHostAlloc(&p, bytes ? bytes : 1, cudaHostAllocPortable);
  if (e != cudaSuccess) {
    cudaGetLastError();
    return fail(e == cudaErrorMemoryAllocation ? FGPU_ERR_OOM : FGPU_ERR_CUDA, std::string("cudaHostAlloc: ") + cudaGetErrorString(e));
  }
  *out = p;
  return FGPU_OK;
  API_CATCH
}

int32_t fgpu_host_free(void* p) {
  API_TRY
  if (p) cudaFreeHost(p);
  return FGPU_OK;
  API_CATCH
}

int32_t fgpu_dict_export(fgpu_ctx* ctx, const char* table, const char* column, uint8_t* buf, uint64_t cap,
                         uint64_t* out_len, uint32_t* out_count) {
  API_TRY
  if (!ctx || !table || !column || !out_len || !out_count) return fail(FGPU_ERR_INVALID, "null argument");
  std::lock_guard<std::mutex> lk(ctx->mu);
  auto it = ctx->tables.find(table);
  *out_len = 0;
  *out_count = 0;
  if (it == ctx->tables.end()) return FGPU_OK;
  auto dit = it->second.dicts.find(column);
  if (dit == it->second.dicts.end()) return FGPU_OK;
  if (!write_dict_blob(dit->second.values, buf, cap, out_len, out_count)) return fail(FGPU_ERR_INVALID, "buffer too small");
  return FGPU_OK;
  API_CATCH
}

int32_t fgpu_dict_preload(fgpu_ctx* ctx, const char* table, const char* column, const uint8_t* blob, uint64_t len, uint32_t count) {
  API_TRY
  if (!ctx || !table || !column || (!blob && len)) return fail(FGPU_ERR_INVALID, "null argument");
  std::lock_guard<std::mutex> lk(ctx->mu);
  GlobalDict& d = ctx->tables[table].dicts[column];
  d.preloaded = true;
  const uint8_t* p = blob;
  const uint8_t* end = blob + len;
  for (uint32_t i = 0; i < count; i++) {
    if (end - p < 4) return fail(FGPU_ERR_INVALID, "dictionary blob truncated");
    uint32_t l;
    std::memcpy(&l, p, 4);
    p += 4;
    if (l > uint64_t(end - p)) return fail(FGPU_ERR_INVALID, "dictionary blob truncated");
    d.intern(reinterpret_cast<const char*>(p), l);
    p += l;
  }
  ctx->tables[table].epoch = ++ctx->epoch_counter;
  return FGPU_OK;
  API_CATCH
}

int32_t fgpu_parquet_dict_values(const uint8_t* file, uint64_t len, const char* column, uint8_t* buf, uint64_t cap, uint64_t* out_len,
                                 uint32_t* out_count) {
  API_TRY
  if (!file || !column || !out_len || !out_count) return fail(FGPU_ERR_INVALID, "null argument");
  ParsedFile pf;
  std::string err;
  if (!parse_parquet(file, len, &pf, &err)) return fail(FGPU_ERR_PARQUET, err);
  GlobalDict d;  // first-seen order over the file's row groups
  if (!column_dict_values(pf, column, &d, &err)) return fail(FGPU_ERR_PARQUET, err);
  if (!write_dict_blob(d.values, buf, cap, out_len, out_count)) return fail(FGPU_ERR_INVALID, "buffer too small");
  return FGPU_OK;
  API_CATCH
}

int32_t fgpu_part_decode_column(fgpu_ctx* ctx, const char* table, uint64_t part_id, const char* column,
                                struct ArrowSchema* out_schema, struct ArrowArray* out_array) {
  API_TRY
  if (!ctx || !table || !column || !out_schema || !out_array) return fail(FGPU_ERR_INVALID, "null argument");
  std::lock_guard<std::mutex> lk(ctx->mu);
  CUDA_TRY(cudaSetDevice(ctx->device));
  auto it = ctx->tables.find(table);
  if (it == ctx->tables.end()) return fail(FGPU_ERR_NOT_FOUND, std::string("table not found: ") + table);
  Part* part = nullptr;
  for (auto& p : it->second.parts)
    if (p->id == part_id) part = p.get();
  if (!part) return fail(FGPU_ERR_NOT_FOUND, "part not found");
  {
    UploadStats st;
    int32_t rc = upload_columns(ctx, &it->second, {{part, column}}, &st, /*refuse_unreadable=*/false);
    if (rc) return rc;
    const ColumnImage& img = part->images[column];
    if (!img.error.empty() && img.error != "column not in part") return fail(FGPU_ERR_UNSUPPORTED, std::string(column) + ": " + img.error);
  }
  uint64_t total = 0;
  int phys = -1;
  for (auto& rg : part->rgs) {
    auto c = rg.cols.find(column);
    if (c == rg.cols.end()) return fail(FGPU_ERR_NOT_FOUND, std::string("column not found: ") + column);
    if (!c->second.error.empty()) return fail(FGPU_ERR_UNSUPPORTED, std::string(column) + ": " + c->second.error);
    phys = c->second.phys;
    total += rg.n_rows;
  }
  const bool is_str = phys == PT_BYTE_ARRAY;
  DevBuf d_vals, d_valid;
  CUDA_TRY(d_vals.alloc(total * (is_str ? 4 : 8), ctx->stream));
  if (!is_str) CUDA_TRY(d_valid.alloc(total, ctx->stream));
  uint64_t row = 0;
  for (auto& rg : part->rgs) {
    const ChunkDesc& cd = rg.cols.at(column).desc;
    CUDA_TRY(launch_decode(cd, is_str ? static_cast<int32_t*>(d_vals.p) + row : nullptr,
                           is_str ? nullptr : static_cast<long long*>(d_vals.p) + row,
                           is_str ? nullptr : static_cast<uint8_t*>(d_valid.p) + row, ctx->sm_count, ctx->stream));
    row += rg.n_rows;
  }
  OwnedColumn col;
  col.name = column;
  col.length = int64_t(total);
  if (is_str) {
    std::vector<int32_t> ids(total);
    CUDA_TRY(cudaMemcpyAsync(ids.data(), d_vals.p, total * 4, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    dict_key_column(col, ids.data(), total, nullptr, it->second.dicts.at(column).values, KeyDict::kWhole);
  } else {
    col.format = phys == PT_DOUBLE ? "g" : "l";
    col.data.resize(total * 8);
    std::vector<uint8_t> valid(total);
    CUDA_TRY(cudaMemcpyAsync(col.data.data(), d_vals.p, total * 8, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(cudaMemcpyAsync(valid.data(), d_valid.p, total, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    validity_from_bytes(col, valid.data(), total);
  }
  release_staging(ctx);
  export_column(std::move(col), out_schema, out_array);
  return FGPU_OK;
  API_CATCH
}

int32_t fgpu_parquet_describe(const uint8_t* file, uint64_t len, int32_t tile_rows, char* buf, uint64_t cap,
                              uint64_t* out_len) {
  API_TRY
  if (!file || !out_len) return fail(FGPU_ERR_INVALID, "null argument");
  if (tile_rows == 0) tile_rows = kTileRows;
  if (tile_rows != kTileRows) return fail(FGPU_ERR_INVALID, "tile_rows must be 0 (default)");
  std::string err;
  std::string js = describe_part_json(file, len, kIndexRows, &err);
  if (js.empty()) return fail(FGPU_ERR_PARQUET, err);
  *out_len = js.size();
  if (!buf) return FGPU_OK;
  if (cap < js.size()) return fail(FGPU_ERR_INVALID, "buffer too small");
  std::memcpy(buf, js.data(), js.size());
  return FGPU_OK;
  API_CATCH
}

}  // extern "C"
