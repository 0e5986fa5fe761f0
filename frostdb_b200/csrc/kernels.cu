// sm_90a kernels of libfrostgpu.
//
//   k_scan       K1+K2+K4/K5 fused.  Every warp walks the stored Parquet encodings of the projected column
//                chunks (PLAIN int64/double, RLE/bit-packed hybrid definition levels and dictionary
//                indices) with per-lane run cursors seeded from a per-128-row seed, evaluates the
//                predicate leaves, and folds the selected rows into the aggregate table.
//                Rows whose group does not change inside a warp (the common case for parts sorted in
//                compaction order) are accumulated in registers and flushed with ONE warp-reduced
//                atomic per aggregate when the group changes; mixed groups fall back to
//                __match_any_sync peer reduction.  Replaces ParquetConverter.Convert
//                (pqarrow/arrow.go:264-373), PredicateFilter.Callback (filter.go:255-323),
//                HashAggregate.Callback (aggregate.go:263-490), Distinction.Callback (distinct.go:70-170).
//   k_rows       K1+K2+K3: same decode + predicate, then order-preserving stream compaction
//                (warp ballot + decoupled look-back prefix over tiles) of the projected columns:
//                PredicateFilter.filter() (filter.go:276-323) + Projection.
//   k_finalize   K6: aggregate table -> compacted result columns (finishAggregate, aggregate.go:543-633).
//   k_merge      K6: folds gathered partial tables into the local one (Synchronizer + final
//                HashAggregate, synchronize.go:16-53, physicalplan.go:438-471).
//   k_decode     K1 standalone: one column chunk -> dense buffers.
//   k_flatten    dictionary column chunk -> flat code array for the tile kernel (tile_agg.cu).
//
// Every general kernel (k_scan, k_rows, k_decode, k_flatten) reads the hybrid streams of a column chunk through one
// pair of readers, DictReader and NumReader, 32 rows per step from the per-128-row seeds: k_scan seeds them from its
// vector's ring slot, the others from the chunk's global seeds.
//
// HBM-bound integer / indexing work: no tensor cores.  k_scan is a vectorized engine: every warp owns
// vectors of 512 rows, prefetches the vector's PLAIN column slices and hybrid-stream seeds into a
// private shared-memory ring with 16-byte cp.async (LDGSTS) groups two vectors ahead, and runs either
// a fused register-only pass (conjunctive range filter + dense dictionary keys + Sum/Min/Max/Count) or
// a general column-at-a-time path with per-row intermediates in shared memory.  (A cp.async.bulk/TMA
// ring was tried first: 2 KB bulk copies per warp were slower, the bulk-copy engine is the wrong tool for
// per-warp vectors; see DESIGN.md.)
#include <cuda_runtime.h>

#include <algorithm>
#include <climits>
#include <cstdint>
#include <map>
#include <mutex>

#include "device_types.h"
#include "kernels.h"
#include "agg_ops.cuh"
#include "ptx.cuh"

namespace fgpu {

namespace {

constexpr int NT = kScanThreads;     // threads per CTA
constexpr int NWARP = NT / 32;       // warps per CTA = chunks per tile
constexpr int STEPS = kIndexRows / 32;  // 32-row steps per chunk
static_assert(NWARP * kIndexRows == kTileRows, "k_rows: tile = one chunk per warp");
static_assert(STEPS == 4, "unrolled for 4 steps");

constexpr uint32_t kNoSlot = 0xffffffffu;
constexpr uint32_t FULL = 0xffffffffu;

// ---- hybrid stream cursor ------------------------------------------------------------------------------
struct HybCur {
  const Run* runs;
  const uint8_t* stream;
  const uint32_t* lut;  // string dictionaries: bit-packed index -> global id (RLE values are global ids already)
  uint32_t k, start, end, val, meta, off;
};

__device__ __forceinline__ void hc_load(HybCur& c) {
  uint4 r = __ldg(reinterpret_cast<const uint4*>(c.runs + c.k));
  c.start = r.x;
  c.off = r.y;
  c.val = r.z;
  c.meta = r.w;
  c.end = __ldg(&c.runs[c.k + 1].start);
}
// `seed` may live in shared memory (staged by the producer) or in global memory.
__device__ __forceinline__ uint32_t hc_init(HybCur& c, const Run* runs, const uint8_t* stream, const uint32_t* lut, const Seed* seed) {
  const uint4 a = *reinterpret_cast<const uint4*>(seed);
  const uint4 b = *(reinterpret_cast<const uint4*>(seed) + 1);
  c.runs = runs;
  c.stream = stream;
  c.lut = lut;
  c.k = a.x;
  c.start = a.y;
  c.end = a.z;
  c.off = a.w;
  c.val = b.x;
  c.meta = b.y;
  return b.z;  // val0
}
__device__ __forceinline__ uint32_t extract_bits(const uint8_t* stream, uint32_t off, uint64_t bit, uint32_t w) {
  uint64_t byte = uint64_t(off) + (bit >> 3);
  const uint32_t* wp = reinterpret_cast<const uint32_t*>(stream) + (byte >> 2);
  uint32_t sh = uint32_t(byte & 3) * 8 + uint32_t(bit & 7);
  uint32_t lo = __ldg(wp), hi = __ldg(wp + 1);
  uint32_t v = __funnelshift_r(lo, hi, sh);
  uint32_t mask = (w >= 32) ? 0xffffffffu : ((1u << w) - 1u);
  return v & mask;
}
// Value at ordinal `ord` (ordinals are requested in increasing order per lane).
__device__ __forceinline__ uint32_t hc_get(HybCur& c, uint32_t ord) {
  while (ord >= c.end) {
    c.k++;
    hc_load(c);
  }
  if ((c.meta & 1u) == 0) return c.val;
  uint32_t w = (c.meta >> 8) & 0xffu;
  uint32_t v = extract_bits(c.stream, c.off, uint64_t(ord - c.start) * w, w);
  return c.lut ? __ldg(c.lut + v) : v;
}

// ---- predicate --------------------------------------------------------------------------------------------
// Canonical numeric leaf: value inside [lo, hi] (inclusive), optionally negated.  NaN is never inside.
__device__ __forceinline__ bool leaf_range(const LeafDesc& ld, long long bits, bool f64col) {
  bool in;
  if (ld.cmp_float) {
    const double x = f64col ? __longlong_as_double(bits) : double(bits);
    in = x >= ld.lo_f && x <= ld.hi_f;
  } else {
    in = bits >= ld.lo_i && bits <= ld.hi_i;
  }
  return in != (ld.neg != 0);
}

// A postfix program over leaf bits (0..31 push leaf; 0x80 AND; 0x81 OR): the filter's and each boolean key's.
__device__ __forceinline__ bool eval_postfix(const uint8_t* prog, int n, uint32_t bits) {
  uint32_t stack = 0;  // stack kept in a 32-bit word
  int sp = 0;
  for (int i = 0; i < n; i++) {
    uint8_t op = prog[i];
    if (op < 0x80) {
      stack = (stack & ~(1u << sp)) | (((bits >> op) & 1u) << sp);
      sp++;
    } else {
      uint32_t b = (stack >> (sp - 1)) & 1u, a = (stack >> (sp - 2)) & 1u;
      uint32_t r = (op == 0x80) ? (a & b) : (a | b);
      sp -= 2;
      stack = (stack & ~(1u << sp)) | (r << sp);
      sp++;
    }
  }
  return stack & 1u;
}

__device__ __forceinline__ bool eval_filter(const QueryDesc& q, uint32_t bits) {
  if (q.filter_kind == FK_AND) return (bits & q.filter_mask) == q.filter_mask;
  if (q.filter_kind == FK_OR) return (bits & q.filter_mask) != 0;
  return eval_postfix(q.filter_prog, q.n_filter_prog, bits);
}

// ---- aggregate expressions ----------------------------------------------------------------------------------
// Arithmetic ignores validity and Div by zero yields NULL, i.e. a raw 0 in the aggregated array
// (query/physicalplan/project.go:169-395, :216-218).
__device__ __forceinline__ long long apply_arith(uint8_t op, bool is_float, long long lb, long long rb) {
  if (is_float) {
    double l = __longlong_as_double(lb), r = __longlong_as_double(rb), x;
    switch (op) {
      case PO_ADD: x = l + r; break;
      case PO_SUB: x = l - r; break;
      case PO_MUL: x = l * r; break;
      default: x = (r == 0.0) ? 0.0 : l / r; break;
    }
    return __double_as_longlong(x);
  }
  unsigned long long l = (unsigned long long)lb, r = (unsigned long long)rb;
  switch (op) {
    case PO_ADD: return (long long)(l + r);
    case PO_SUB: return (long long)(l - r);
    case PO_MUL: return (long long)(l * r);
    default:
      if (rb == 0) return 0;
      if (rb == -1) return (long long)(0ull - l);  // Go wraps INT64_MIN / -1
      return lb / rb;
  }
}

// ---- aggregate table ----------------------------------------------------------------------------------------
__device__ __forceinline__ uint64_t mix64(uint64_t x) {
  x ^= x >> 33;
  x *= 0xff51afd7ed558ccdull;
  x ^= x >> 33;
  x *= 0xc4ceb9fe1a85ec53ull;
  x ^= x >> 33;
  return x;
}

// Exact-key open addressing: a slot is claimed by CAS on its tag (0 -> 1), the key words are
// written, then the tag is published as fingerprint|2.  Unlike the reference, which keys groups
// only by a 64-bit hash (aggregate.go:411), equal tags are confirmed against the stored key.
template <int KW>
__device__ __forceinline__ uint32_t hash_find_or_insert(const QueryDesc& q, const unsigned long long (&kw)[KW], bool* overflow) {
  const int W = q.key_words;
  uint64_t h = 0x9e3779b97f4a7c15ull;
#pragma unroll
  for (int w = 0; w < KW; w++)
    if (w < W) h = mix64(h ^ kw[w]) + 0x9e3779b97f4a7c15ull * (w + 1);
  const uint32_t fp = uint32_t(h >> 32) | 2u;
  const uint32_t mask = q.table_slots - 1;
  uint32_t s = uint32_t(h) & mask;
  volatile uint32_t* tag = q.t_tag;
  volatile unsigned long long* keys = q.t_keys;
  for (uint32_t probes = 0; probes <= mask; probes++) {
    uint32_t t = tag[s];
    if (t == 0) {
      uint32_t old = atomicCAS(q.t_tag + s, 0u, 1u);
      if (old == 0) {
#pragma unroll
        for (int w = 0; w < KW; w++)
          if (w < W) keys[size_t(s) * W + w] = kw[w];
        __threadfence();
        tag[s] = fp;
        return s;
      }
      t = old;
    }
    while (t == 1u) t = tag[s];
    if (t == fp) {
      bool eq = true;
#pragma unroll
      for (int w = 0; w < KW; w++)
        if (w < W) eq &= (keys[size_t(s) * W + w] == kw[w]);
      if (eq) return s;
    }
    s = (s + 1) & mask;
  }
  *overflow = true;
  return 0;
}

template <typename T, typename Op>
__device__ __forceinline__ T warp_reduce(T v, Op op) {
#pragma unroll
  for (int d = 16; d >= 1; d >>= 1) v = op(v, __shfl_xor_sync(FULL, v, d));
  return v;
}

template <typename T, typename Op>
__device__ __forceinline__ T peer_reduce(T v, unsigned peers, int lane, Op op) {
  const int cnt = __popc(peers);
  if (cnt == 1) return v;
  const int rank = __popc(peers & ((1u << lane) - 1u));
  for (int stride = 1; stride < cnt; stride <<= 1) {
    int srcrank = rank + stride;
    int src = (srcrank < cnt) ? int(__fns(peers, 0, srcrank + 1)) : lane;
    T o = __shfl_sync(peers, v, src);
    if (srcrank < cnt && (rank & (2 * stride - 1)) == 0) v = op(v, o);
  }
  return v;  // valid in the lowest lane of the peer group
}

// Warp-reduces the per-lane partial of one aggregate and lets lane 0 apply it to the table cell.
__device__ __noinline__ void flush_agg(uint8_t func, bool is_float, long long* cell, long long acc, int lane) {
  acc = warp_reduce(acc, [=](long long a, long long b) { return agg_combine(func, is_float, a, b); });
  if (lane == 0) apply_agg(func, is_float, cell, acc);
}

// One step whose active lanes belong to different groups.  Sorted parts put at most a few groups in one
// 32-row step (a run boundary), so the groups are peeled off one at a time with masked full-warp
// reductions; only steps with more than 4 groups fall back to __match_any_sync peer reduction.
__device__ __noinline__ void mixed_agg(uint8_t func, bool is_float, long long* column, uint32_t slot, bool active, long long bits,
                                       int lane) {
  unsigned remaining = __ballot_sync(FULL, active);
  const long long ident = agg_identity(func, is_float);
  for (int round = 0; round < 4 && remaining; round++) {
    const uint32_t s0 = __shfl_sync(FULL, slot, __ffs(remaining) - 1);
    const bool mine = active && slot == s0;
    long long v = mine ? bits : ident;
    v = warp_reduce(v, [=](long long a, long long b) { return agg_combine(func, is_float, a, b); });
    if (lane == 0) apply_agg(func, is_float, column + s0, v);
    remaining &= ~__ballot_sync(FULL, mine);
  }
  if (remaining == 0) return;
  const bool left = (remaining >> lane) & 1u;
  if (!left) return;
  unsigned peers = __match_any_sync(remaining, slot);
  long long r = peer_reduce(bits, peers, lane, [=](long long a, long long b) { return agg_combine(func, is_float, a, b); });
  if (lane == __ffs(peers) - 1) apply_agg(func, is_float, column + slot, r);
}
__device__ __noinline__ void mixed_rows(unsigned long long* rows, uint32_t slot, bool active, int lane) {
  unsigned remaining = __ballot_sync(FULL, active);
  for (int round = 0; round < 4 && remaining; round++) {
    const uint32_t s0 = __shfl_sync(FULL, slot, __ffs(remaining) - 1);
    const unsigned grp = __ballot_sync(FULL, active && slot == s0);
    if (lane == 0) atomicAdd(rows + s0, (unsigned long long)__popc(grp));
    remaining &= ~grp;
  }
  if (remaining == 0) return;
  const bool left = (remaining >> lane) & 1u;
  if (!left) return;
  unsigned peers = __match_any_sync(remaining, slot);
  if (lane == __ffs(peers) - 1) atomicAdd(rows + slot, (unsigned long long)__popc(peers));
}

// Locates the row group of a tile (rg_first_tile ascending, n_rg + 1 entries).
__device__ __forceinline__ int find_rg(const uint32_t* __restrict__ first_tile, int n_rg, uint32_t tile) {
  int lo = 0, hi = n_rg;
  while (hi - lo > 1) {
    int mid = (lo + hi) >> 1;
    if (__ldg(&first_tile[mid]) <= tile) lo = mid; else hi = mid;
  }
  return lo;
}

}  // namespace

// ======================================================================================================
// k_scan — vectorized, warp-private execution
// ======================================================================================================
// Every warp owns vectors of q.vl rows (128..512, a multiple of 128) of one row group and works through
// them column at a time, like a vectorized CPU engine works through cache-resident vectors: per-row
// intermediates (selection bits, table slot, packed key words, expression temporaries) live in the
// warp's private shared-memory region, so the only per-lane state is the cursor of the ONE column
// being decoded.  The fixed cost of resolving a column (descriptor, seeds, staging) is paid once per
// vector instead of once per 128 rows, which is what made the previous version instruction bound.
// Lane 0 of the warp keeps a private ring of q.n_ring slots filled with cp.async.bulk copies (TMA)
// of the vector's PLAIN column slices and hybrid-stream seeds, issued n_ring-1 vectors ahead.

struct VecCtx {
  const QueryDesc* q;
  const ChunkDesc* chunks;  // [n_slots] of the row group
  const LeafRt* lrt;        // [n_leaves]
  const uint8_t* slotmem;   // ring slot of this vector (PLAIN slices, then seeds)
  uint32_t r0;              // first row of the vector inside the row group
  uint32_t n_rows;          // rows of the row group
  uint32_t chunk;           // index of the vector's first 128-row chunk inside the row group
  int steps;                // 32-row steps in this vector
};

// Streams the rows of one dictionary-encoded string column through the vector: next() must be called by
// all lanes, once per step, in step order.
struct DictReader {
  HybCur vc, dc;
  uint32_t vbase, lt;
  bool absent, nulls;
  __device__ __forceinline__ void init(const VecCtx& v, int slot, int lane) {
    const ChunkDesc& c = v.chunks[slot];
    absent = c.kind == CK_ABSENT;
    nulls = !absent && c.has_nulls;
    lt = (1u << lane) - 1u;
    vbase = v.r0;
    if (absent) return;
    const uint8_t* seeds = v.slotmem + size_t(v.q->n_stage_plain) * v.q->vl * 8;
    const int sv = v.q->slot_seed_stage[slot][0], sd = v.q->slot_seed_stage[slot][1];
    if (nulls) vbase = hc_init(dc, c.def_runs, c.def, nullptr, sd >= 0 ? reinterpret_cast<const Seed*>(seeds) + sd : c.def_seeds + v.chunk);
    hc_init(vc, c.runs, c.values, c.lut, sv >= 0 ? reinterpret_cast<const Seed*>(seeds) + sv : c.seeds + v.chunk);
  }
  // Streams 128-row chunk `chunk` of c from its global seeds.  A second initialiser rather than a core shared with the
  // one above: routing k_scan's through a shared core moves spills across k_scan's call graph.  It starts from a zeroed
  // reader: a cursor the chunk's kind leaves unset would be read undefined across the unrolled steps of the kernels
  // that use it, which keeps its registers live through the whole kernel (k_rows: 151 registers instead of 72).
  __device__ __forceinline__ void init(const ChunkDesc& c, uint32_t chunk, int lane) {
    *this = DictReader{};
    absent = c.kind == CK_ABSENT;
    nulls = !absent && c.has_nulls;
    lt = (1u << lane) - 1u;
    vbase = chunk * kIndexRows;
    if (absent) return;
    if (nulls) vbase = hc_init(dc, c.def_runs, c.def, nullptr, c.def_seeds + chunk);
    hc_init(vc, c.runs, c.values, c.lut, c.seeds + chunk);
  }
  // global dictionary id of row r (this lane's row of the current step), kNullIdx for NULL / out of range
  __device__ __forceinline__ uint32_t next(uint32_t r, uint32_t n_rows) {
    if (absent) return kNullIdx;
    bool valid = r < n_rows;
    uint32_t ord = r;
    if (nulls) {
      if (valid) valid = hc_get(dc, r) != 0;
      unsigned m = __ballot_sync(FULL, valid);
      ord = vbase + __popc(m & lt);
      vbase += __popc(m);
    }
    return valid ? hc_get(vc, ord) : kNullIdx;
  }
};

// Same for a numeric column: raw 8 bytes per row (0 for NULL) + null flag.
struct NumReader {
  HybCur vc, dc;
  const long long* staged;  // shared-memory slice indexed by (row - r0), or nullptr
  const long long* vals;
  const long long* dict64;
  uint32_t vbase, lt, r0;
  uint8_t mode;  // 0 absent, 1 plain direct (staged or global), 2 cursor path
  bool nulls, dict;
  __device__ __forceinline__ void init(const VecCtx& v, int slot, int lane) {
    const ChunkDesc& c = v.chunks[slot];
    r0 = v.r0;
    lt = (1u << lane) - 1u;
    staged = nullptr;
    if (c.kind == CK_ABSENT) { mode = 0; return; }
    vals = reinterpret_cast<const long long*>(c.values);
    if (c.kind == CK_PLAIN64 && !c.has_nulls) {
      mode = 1;
      const int p = v.q->slot_plain_stage[slot];
      if (p >= 0) staged = reinterpret_cast<const long long*>(v.slotmem + size_t(p) * v.q->vl * 8);
      return;
    }
    mode = 2;
    nulls = c.has_nulls;
    dict = c.kind == CK_DICT64;
    dict64 = reinterpret_cast<const long long*>(c.dict64);
    vbase = v.r0;
    const uint8_t* seeds = v.slotmem + size_t(v.q->n_stage_plain) * v.q->vl * 8;
    const int sv = v.q->slot_seed_stage[slot][0], sd = v.q->slot_seed_stage[slot][1];
    if (nulls) vbase = hc_init(dc, c.def_runs, c.def, nullptr, sd >= 0 ? reinterpret_cast<const Seed*>(seeds) + sd : c.def_seeds + v.chunk);
    if (dict) hc_init(vc, c.runs, c.values, nullptr, sv >= 0 ? reinterpret_cast<const Seed*>(seeds) + sv : c.seeds + v.chunk);
  }
  // Streams 128-row chunk `chunk` of c from its global seeds, from a zeroed reader (see DictReader).
  __device__ __forceinline__ void init(const ChunkDesc& c, uint32_t chunk, int lane) {
    *this = NumReader{};
    r0 = chunk * kIndexRows;
    lt = (1u << lane) - 1u;
    if (c.kind == CK_ABSENT) { mode = 0; return; }
    vals = reinterpret_cast<const long long*>(c.values);
    if (c.kind == CK_PLAIN64 && !c.has_nulls) { mode = 1; return; }
    mode = 2;
    nulls = c.has_nulls;
    dict = c.kind == CK_DICT64;
    dict64 = reinterpret_cast<const long long*>(c.dict64);
    vbase = r0;
    if (nulls) vbase = hc_init(dc, c.def_runs, c.def, nullptr, c.def_seeds + chunk);
    if (dict) hc_init(vc, c.runs, c.values, nullptr, c.seeds + chunk);
  }
  __device__ __forceinline__ long long next(uint32_t r, uint32_t n_rows, bool& null) {
    if (mode == 1) {
      null = r >= n_rows;
      if (null) return 0;
      return staged ? staged[r - r0] : __ldg(vals + r);
    }
    if (mode == 0) { null = true; return 0; }
    bool valid = r < n_rows;
    uint32_t ord = r;
    if (nulls) {
      if (valid) valid = hc_get(dc, r) != 0;
      unsigned m = __ballot_sync(FULL, valid);
      ord = vbase + __popc(m & lt);
      vbase += __popc(m);
    }
    null = !valid;
    if (!valid) return 0;
    return dict ? __ldg(dict64 + hc_get(vc, ord)) : __ldg(vals + ord);
  }
};

struct FastPlan;
// Per-warp shared-memory region (offsets precomputed by the host in QueryDesc.wr_*).
struct WarpMem {
  uint64_t* full;            // [n_ring] mbarriers
  uint8_t* ring;             // [n_ring][slot_bytes]
  uint32_t* act;             // [vl/32] selection ballot per step
  uint32_t* leafw;           // [vl] per-row leaf bits (FK_PROGRAM only)
  uint32_t* slotv;           // [vl] table slot per row
  unsigned long long* keyw;  // [key_words][vl] packed key words (hash mode)
  long long* tmp1;           // [vl] expression temporaries
  long long* tmp2;
  long long* acc;            // [kMaxAggs][32] per-lane partial of every aggregate
  unsigned long long* lastkw;  // [kMaxKeyWords][32] hash mode: last key of each lane ...
  uint32_t* lastslot;        // [32] ... and its slot
  uint32_t* cnt;             // [32] per-lane pending row count of the running group
  unsigned long long* selected;  // [1] selected rows seen by this warp
  ChunkDesc* cdesc;          // [n_slots] descriptors of the row group the warp is working on
  LeafRt* clrt;              // [n_leaves]
  struct FastPlan* fplan;    // resolved fast-path plan of that row group
};

__device__ __forceinline__ WarpMem warp_mem(const QueryDesc& q, uint8_t* base) {
  WarpMem m;
  m.full = reinterpret_cast<uint64_t*>(base);
  m.ring = base + q.wr_ring;
  m.act = reinterpret_cast<uint32_t*>(base + q.wr_act);
  m.leafw = reinterpret_cast<uint32_t*>(base + q.wr_leaf);
  m.slotv = reinterpret_cast<uint32_t*>(base + q.wr_slot);
  m.keyw = reinterpret_cast<unsigned long long*>(base + q.wr_keyw);
  m.tmp1 = reinterpret_cast<long long*>(base + q.wr_tmp1);
  m.tmp2 = reinterpret_cast<long long*>(base + q.wr_tmp2);
  m.acc = reinterpret_cast<long long*>(base + q.wr_acc);
  m.selected = reinterpret_cast<unsigned long long*>(base + q.wr_acc + size_t(q.n_aggs) * 32 * 8);
  m.cnt = reinterpret_cast<uint32_t*>(m.selected + 2);
  m.lastslot = m.cnt + 32;
  m.lastkw = reinterpret_cast<unsigned long long*>(m.lastslot + 32);  // [key_words][32], hash mode only
  m.cdesc = reinterpret_cast<ChunkDesc*>(base + q.wr_cdesc);
  m.clrt = reinterpret_cast<LeafRt*>(base + q.wr_clrt);
  m.fplan = reinterpret_cast<struct FastPlan*>(base + q.wr_fplan);
  return m;
}

// All lanes: fill ring slot `rs` with vector `vec` of row group `rg` using 16-byte cp.async (LDGSTS):
// 512 contiguous bytes per warp instruction, no per-copy engine overhead (a per-warp ring of 2 KB
// cp.async.bulk copies was slower).
__device__ __forceinline__ void cp_async16(uint32_t dst_saddr, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst_saddr), "l"(src) : "memory");
}
__device__ __forceinline__ void issue_vector(const QueryDesc& q, uint8_t* ring, uint32_t vec, int rs, uint32_t rg_first, uint32_t n_rows,
                                             const ChunkDesc* chunks, int lane) {
  const uint32_t vec_in_rg = vec - rg_first;
  const uint32_t r0 = vec_in_rg * q.vl;
  const uint32_t n = min(uint32_t(q.vl), n_rows - r0);
  const uint32_t chunk = r0 / kIndexRows;
  const uint32_t dst = smem_u32(ring + size_t(rs) * q.slot_bytes);
  const uint32_t plain_sz = (n * 8u + 15u) & ~15u;
  for (int p = 0; p < q.n_stage_plain; p++) {
    const ChunkDesc& c = chunks[q.stage_plain_slot[p]];
    if (c.kind != CK_PLAIN64 || c.has_nulls) continue;
    const uint8_t* src = c.values + size_t(r0) * 8;
    const uint32_t d = dst + uint32_t(p) * uint32_t(q.vl) * 8u;
    for (uint32_t o = uint32_t(lane) * 16u; o < plain_sz; o += 512u) cp_async16(d + o, src + o);
  }
  const uint32_t seed_base = dst + uint32_t(q.n_stage_plain) * uint32_t(q.vl) * 8u;
  for (int t = 0; t < q.n_stage_seeds; t++) {
    const ChunkDesc& c = chunks[q.stage_seed_slot[t]];
    const bool is_def = q.stage_seed_is_def[t];
    const bool present = is_def ? (c.kind != CK_ABSENT && c.has_nulls) : (c.kind == CK_DICT_STR || c.kind == CK_DICT64);
    if (present && lane < 2)
      cp_async16(seed_base + uint32_t(t) * uint32_t(sizeof(Seed)) + uint32_t(lane) * 16u,
                 reinterpret_cast<const uint8_t*>((is_def ? c.def_seeds : c.seeds) + chunk) + lane * 16);
  }
  asm volatile("cp.async.commit_group;" ::: "memory");
}
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

// ---- selection -------------------------------------------------------------------------------------------
// act[s] = ballot over the 32 rows of step s that pass the predicate.
__device__ __noinline__ uint32_t vec_selection(const VecCtx& v, uint8_t* wb, int lane) {
  const WarpMem m = warp_mem(*v.q, wb);
  const QueryDesc& q = *v.q;
  const int steps = v.steps;
  for (int s = lane; s < steps; s += 32) {
    const uint32_t first = v.r0 + uint32_t(s) * 32;
    const uint32_t left = v.n_rows > first ? v.n_rows - first : 0;
    m.act[s] = left >= 32 ? FULL : ((1u << left) - 1u);  // rows inside the row group
  }
  __syncwarp();
  if (q.n_filter_prog == 0) {
    uint32_t any = 0;
    #pragma unroll 1
    for (int s = 0; s < steps; s++) any |= m.act[s];
    return any;
  }
  const bool prog = q.filter_kind == FK_PROGRAM;
  const bool is_or = q.filter_kind == FK_OR;
  if (prog) {
    for (int i = lane; i < q.vl; i += 32) m.leafw[i] = 0;
  } else if (is_or) {
    // disjunction: start from nothing selected, remember the in-range mask in leafw
    for (int s = lane; s < steps; s += 32) {
      m.leafw[s] = m.act[s];
      m.act[s] = 0;
    }
  }
  __syncwarp();
  for (int l = 0; l < q.n_leaves; l++) {
    const LeafDesc& ld = q.leaves[l];
    const LeafRt& rt = v.lrt[l];
    if (rt.mode != LM_EVAL) {
      const bool all = rt.mode == LM_ALL;
      if (prog) {
        if (all)
          for (int i = lane; i < q.vl; i += 32) m.leafw[i] |= 1u << l;
      } else if (is_or) {
        if (all)
          for (int s = lane; s < steps; s += 32) m.act[s] = m.leafw[s];
      } else if (!all) {
        for (int s = lane; s < steps; s += 32) m.act[s] = 0;
      }
      __syncwarp();
      continue;
    }
    if (q.slot_type[ld.slot] == ST_DICT) {
      DictReader rd;
      rd.init(v, ld.slot, lane);
      const uint8_t* lut = rt.lut;
      const uint32_t nullres = rt.null_result;
      #pragma unroll 1
      for (int s = 0; s < steps; s++) {
        const uint32_t r = v.r0 + uint32_t(s) * 32 + lane;
        const uint32_t gid = rd.next(r, v.n_rows);
        const bool res = r < v.n_rows && ((gid == kNullIdx) ? nullres : uint32_t(__ldg(lut + gid))) != 0;
        if (prog) {
          if (res) m.leafw[s * 32 + lane] |= 1u << l;
        } else {
          const unsigned b = __ballot_sync(FULL, res);
          if (lane == 0) m.act[s] = is_or ? (m.act[s] | b) : (m.act[s] & b);
        }
      }
    } else {
      NumReader rd;
      rd.init(v, ld.slot, lane);
      const bool f64col = q.slot_type[ld.slot] == ST_F64;
#pragma unroll 1
      for (int s = 0; s < steps; s++) {
        const uint32_t r = v.r0 + uint32_t(s) * 32 + lane;
        bool null;
        const long long bits = rd.next(r, v.n_rows, null);
        const bool res = !null && leaf_range(ld, bits, f64col);
        if (prog) {
          if (res) m.leafw[s * 32 + lane] |= 1u << l;
        } else {
          const unsigned b = __ballot_sync(FULL, res);
          if (lane == 0) m.act[s] = is_or ? (m.act[s] | b) : (m.act[s] & b);
        }
      }
    }
    __syncwarp();
  }
  if (prog) {
    #pragma unroll 1
    for (int s = 0; s < steps; s++) {
      const bool res = eval_filter(q, m.leafw[s * 32 + lane]);
      const unsigned b = __ballot_sync(FULL, res);
      if (lane == 0) m.act[s] &= b;
    }
    __syncwarp();
  }
  uint32_t any = 0;
  #pragma unroll 1
  for (int s = 0; s < steps; s++) any |= m.act[s];
  return any;
}

// ---- aggregate input vector -------------------------------------------------------------------------------
// Evaluates an aggregate expression over the vector into out[] (raw 8-byte values, NULL slots 0).
__device__ __noinline__ void vec_eval_expr(const VecCtx& v, uint8_t* wb, const AggDesc& a, int lane, long long* out) {
  const WarpMem m = warp_mem(*v.q, wb);
  const QueryDesc& q = *v.q;
  long long* stack[3] = {out, m.tmp2, m.tmp2 + q.vl};  // operand stack: depth <= 3 (checked by the host)
  int sp = 0;
  for (int p = a.prog_off; p < a.prog_off + a.prog_len; p++) {
    const ProgOp& o = q.prog[p];
    if (o.op == PO_LOAD) {
      NumReader rd;
      rd.init(v, o.slot, lane);
      long long* dst = stack[sp];
      #pragma unroll 1
      for (int s = 0; s < v.steps; s++) {
        bool null;
        dst[s * 32 + lane] = rd.next(v.r0 + uint32_t(s) * 32 + lane, v.n_rows, null);
      }
      sp++;
    } else if (o.op == PO_CONST) {
      long long* dst = stack[sp];
      #pragma unroll 1
      for (int s = 0; s < v.steps; s++) dst[s * 32 + lane] = o.imm;
      sp++;
    } else {
      long long* l = stack[sp - 2];
      const long long* r = stack[sp - 1];
      #pragma unroll 1
      for (int s = 0; s < v.steps; s++) l[s * 32 + lane] = apply_arith(o.op, a.is_float, l[s * 32 + lane], r[s * 32 + lane]);
      sp--;
    }
  }
}

// ---- boolean keys -----------------------------------------------------------------------------------------
// The per-warp copy of the plan's BoolKeys block, followed by the key leaves' LeafRt of the current row group.
__device__ __forceinline__ const BoolKeys& warp_bool_keys(const QueryDesc& q, uint8_t* wb) {
  return *reinterpret_cast<const BoolKeys*>(wb + __ldg(&q.bool_keys->wr_keys));
}

// leafw[row] bit l = key leaf l holds on that row: the filter's leaf rules (vec_selection), so a NULL numeric value is
// false and a dictionary leaf takes null_result.  The selection is done with leafw by now.
__device__ __noinline__ void vec_key_leaves(const VecCtx& v, uint8_t* wb, int lane) {
  const WarpMem m = warp_mem(*v.q, wb);
  const QueryDesc& q = *v.q;
  const BoolKeys& bk = warp_bool_keys(q, wb);
  const LeafRt* klrt = reinterpret_cast<const LeafRt*>(&bk + 1);
  uint32_t cbits = 0;
  for (int l = 0; l < bk.n_leaves; l++)
    if (klrt[l].mode == LM_ALL) cbits |= 1u << l;
  for (int s = 0; s < v.steps; s++) m.leafw[s * 32 + lane] = cbits;
  for (int l = 0; l < bk.n_leaves; l++) {
    const LeafDesc& ld = bk.leaves[l];
    const LeafRt& rt = klrt[l];
    if (rt.mode != LM_EVAL) continue;
    if (q.slot_type[ld.slot] == ST_DICT) {
      DictReader rd;
      rd.init(v, ld.slot, lane);
      const uint8_t* lut = rt.lut;
      const uint32_t nullres = rt.null_result;
#pragma unroll 1
      for (int s = 0; s < v.steps; s++) {
        const uint32_t gid = rd.next(v.r0 + uint32_t(s) * 32 + lane, v.n_rows);
        const uint32_t res = (gid == kNullIdx) ? nullres : uint32_t(__ldg(lut + gid));
        m.leafw[s * 32 + lane] |= (res & 1u) << l;
      }
    } else {
      NumReader rd;
      rd.init(v, ld.slot, lane);
      const bool f64col = q.slot_type[ld.slot] == ST_F64;
#pragma unroll 1
      for (int s = 0; s < v.steps; s++) {
        bool null;
        const long long bits = rd.next(v.r0 + uint32_t(s) * 32 + lane, v.n_rows, null);
        m.leafw[s * 32 + lane] |= uint32_t(!null && leaf_range(ld, bits, f64col)) << l;
      }
    }
  }
  __syncwarp();
}

// Code of a boolean key on this lane's row of step s: 1 false, 2 true, as hashBooleanArray hashes them
// (dynparquet/hashed.go:228-242): neither is the NULL code 0.
__device__ __forceinline__ uint32_t bool_key_code(const BoolKeys& bk, const KeyDesc& kd, const WarpMem& m, int s, int lane) {
  return 1u + uint32_t(eval_postfix(bk.prog + kd.prog_off, kd.prog_len, m.leafw[s * 32 + lane]));
}

// Copies the key leaves' LeafRt of row group rg behind the warp's copy of the BoolKeys block, and the block itself at
// the warp's first row group.
__device__ __noinline__ void load_bool_keys(const QueryDesc& q, uint8_t* wb, int rg, bool first, int lane) {
  uint32_t* dst = reinterpret_cast<uint32_t*>(wb + __ldg(&q.bool_keys->wr_keys));
  if (first) {
    const uint32_t* src = reinterpret_cast<const uint32_t*>(q.bool_keys);
    for (uint32_t i = lane; i < sizeof(BoolKeys) / 4; i += 32) dst[i] = __ldg(src + i);
    __syncwarp();
  }
  const BoolKeys& bk = *reinterpret_cast<const BoolKeys*>(dst);
  const uint32_t* src = reinterpret_cast<const uint32_t*>(bk.leaf_rt + size_t(rg) * bk.n_leaves);
  dst = reinterpret_cast<uint32_t*>(reinterpret_cast<BoolKeys*>(dst) + 1);
  for (uint32_t i = lane; i < uint32_t(bk.n_leaves) * sizeof(LeafRt) / 4; i += 32) dst[i] = __ldg(src + i);
}

// ---- table slot per row ----------------------------------------------------------------------------------
__device__ __noinline__ void vec_slots_dense(const VecCtx& v, uint8_t* wb, int lane) {
  const WarpMem m = warp_mem(*v.q, wb);
  const QueryDesc& q = *v.q;
  bool first = true;
  if (q.bool_keys) vec_key_leaves(v, wb, lane);
  for (int k = 0; k < q.n_keys; k++) {
    const KeyDesc& kd = q.keys[k];
    if (kd.is_bool) {
      const BoolKeys& bk = warp_bool_keys(q, wb);
#pragma unroll 1
      for (int s = 0; s < v.steps; s++) {
        const uint32_t add = bool_key_code(bk, kd, m, s, lane) * kd.dense_stride;
        m.slotv[s * 32 + lane] = first ? add : m.slotv[s * 32 + lane] + add;
      }
      first = false;
      continue;
    }
    DictReader rd;
    rd.init(v, kd.slot, lane);
    const uint32_t stride = kd.dense_stride;
#pragma unroll 1
    for (int s = 0; s < v.steps; s++) {
      const uint32_t gid = rd.next(v.r0 + uint32_t(s) * 32 + lane, v.n_rows);
      const uint32_t add = (gid == kNullIdx) ? 0u : (gid + 1u) * stride;
      m.slotv[s * 32 + lane] = first ? add : m.slotv[s * 32 + lane] + add;
    }
    first = false;
  }
  if (first)
    for (int s = 0; s < v.steps; s++) m.slotv[s * 32 + lane] = 0;  // no keys: one global group
  __syncwarp();
}

// Hash mode: packed key words per row in shared memory, then find-or-insert (with a per-lane
// last-key cache in m.lastkw: sorted parts repeat the previous row's key most of the time).
__device__ __noinline__ bool vec_slots_hash(const VecCtx& v, uint8_t* wb, int lane) {
  const WarpMem m = warp_mem(*v.q, wb);
  const QueryDesc& q = *v.q;
  const int W = q.key_words;
  bool overflow = false;
  for (int w = 0; w < W; w++)
    for (int s = 0; s < v.steps; s++) m.keyw[size_t(w) * q.vl + s * 32 + lane] = 0;
  if (q.bool_keys) vec_key_leaves(v, wb, lane);
  for (int k = 0; k < q.n_keys; k++) {
    const KeyDesc& kd = q.keys[k];
    unsigned long long* kwp = m.keyw + size_t(kd.word) * q.vl;
    if (kd.is_bool) {
      const BoolKeys& bk = warp_bool_keys(q, wb);
      const uint32_t shift = kd.shift;
#pragma unroll 1
      for (int s = 0; s < v.steps; s++) kwp[s * 32 + lane] |= (unsigned long long)bool_key_code(bk, kd, m, s, lane) << shift;
    } else if (kd.is_int64 && kd.prog_len) {
      // computed key (the sqlparse pre-projection `(timestamp / 1000) * 1000 as bucket`, project.go:58-167): the
      // expression is evaluated into the warp's temporaries; Div by zero yields 0, which groups like NULL
      AggDesc kx{};
      kx.prog_off = kd.prog_off;
      kx.prog_len = kd.prog_len;
      vec_eval_expr(v, wb, kx, lane, m.tmp1);
      __syncwarp();
#pragma unroll 1
      for (int s = 0; s < v.steps; s++) kwp[s * 32 + lane] = (unsigned long long)m.tmp1[s * 32 + lane];
    } else if (kd.is_int64) {
      NumReader rd;
      rd.init(v, kd.slot, lane);
#pragma unroll 1
      for (int s = 0; s < v.steps; s++) {
        bool null;
        // NULL and 0 hash alike in the reference (dynparquet/hashed.go:254-262): NULL slots hold 0
        kwp[s * 32 + lane] = (unsigned long long)rd.next(v.r0 + uint32_t(s) * 32 + lane, v.n_rows, null);
      }
    } else {
      DictReader rd;
      rd.init(v, kd.slot, lane);
      const uint32_t shift = kd.shift;
#pragma unroll 1
      for (int s = 0; s < v.steps; s++) {
        const uint32_t gid = rd.next(v.r0 + uint32_t(s) * 32 + lane, v.n_rows);
        const unsigned long long code = (gid == kNullIdx) ? 0ull : (unsigned long long)gid + 1ull;
        kwp[s * 32 + lane] |= code << shift;
      }
    }
  }
  unsigned long long* lastkw = m.lastkw + lane;  // [kMaxKeyWords][32]
  uint32_t last_slot = m.lastslot[lane];
#pragma unroll 1
  for (int s = 0; s < v.steps; s++) {
    uint32_t sl = kNoSlot;
    if ((m.act[s] >> lane) & 1u) {
      unsigned long long key[kMaxKeyWords];
      bool same = last_slot != kNoSlot;
#pragma unroll
      for (int w = 0; w < kMaxKeyWords; w++) {
        key[w] = (w < W) ? m.keyw[size_t(w) * q.vl + s * 32 + lane] : 0ull;
        same &= (w >= W) || key[w] == lastkw[w * 32];
      }
      if (!same) {
        last_slot = hash_find_or_insert<kMaxKeyWords>(q, key, &overflow);
#pragma unroll
        for (int w = 0; w < kMaxKeyWords; w++)
          if (w < W) lastkw[w * 32] = key[w];
      }
      sl = last_slot;
    }
    m.slotv[s * 32 + lane] = sl;
  }
  m.lastslot[lane] = last_slot;
  __syncwarp();
  return overflow;
}

// ---- rows-per-group counter (also every Count aggregate, aggregate.go:937-950) ------------------------------
// Returns the running group after the vector; m.cnt[lane] carries this lane's pending row count.
__device__ __noinline__ uint32_t vec_count_rows(const VecCtx& v, uint8_t* wb, int lane, uint32_t cur_slot) {
  const WarpMem m = warp_mem(*v.q, wb);
  const QueryDesc& q = *v.q;
  uint32_t cs = cur_slot;
  uint32_t cnt = m.cnt[lane];
  uint32_t selected = 0;
#pragma unroll 1
  for (int s = 0; s < v.steps; s++) {
    const unsigned amask = m.act[s];
    if (amask == 0) continue;
    const bool active = (amask >> lane) & 1u;
    const uint32_t sl = m.slotv[s * 32 + lane];
    selected += __popc(amask);
    const uint32_t s0 = __shfl_sync(FULL, sl, __ffs(amask) - 1);
    const bool uni = __all_sync(FULL, !active || sl == s0);
    if (!uni) {
      if (cs != kNoSlot) {
        const uint32_t tt = __reduce_add_sync(FULL, cnt);
        if (lane == 0 && tt) atomicAdd(q.t_rows + cs, (unsigned long long)tt);
        cnt = 0;
        cs = kNoSlot;
      }
      mixed_rows(q.t_rows, sl, active, lane);
    } else {
      if (s0 != cs) {
        if (cs != kNoSlot) {
          const uint32_t tt = __reduce_add_sync(FULL, cnt);
          if (lane == 0 && tt) atomicAdd(q.t_rows + cs, (unsigned long long)tt);
          cnt = 0;
        }
        cs = s0;
      }
      cnt += active ? 1u : 0u;
    }
  }
  m.cnt[lane] = cnt;
  if (lane == 0) m.selected[0] += selected;
  return cs;
}

// ---- one aggregate over the vector: per-lane partial while the warp stays in one group ------------------------
__device__ __noinline__ void vec_aggregate(const VecCtx& v, uint8_t* wb, int a, int lane, uint32_t cur_slot) {
  const WarpMem m = warp_mem(*v.q, wb);
  const QueryDesc& q = *v.q;
  const AggDesc& ad = q.aggs[a];
  const uint8_t func = ad.func;
  const bool isf = ad.is_float;
  const long long ident = agg_identity(func, isf);
  long long* cells = q.t_agg[a];
  // input: a column read in place, or an expression evaluated into tmp1
  const bool simple = ad.prog_len == 1 && q.prog[ad.prog_off].op == PO_LOAD;
  NumReader rd;
  if (simple) rd.init(v, q.prog[ad.prog_off].slot, lane);
  else vec_eval_expr(v, wb, ad, lane, m.tmp1);
  __syncwarp();
  uint32_t cs = cur_slot;
  long long part = m.acc[a * 32 + lane];
#pragma unroll 1
  for (int s = 0; s < v.steps; s++) {
    long long val;
    if (simple) {
      bool null;
      val = rd.next(v.r0 + uint32_t(s) * 32 + lane, v.n_rows, null);  // every step: the cursor must see all rows
      if (null && ad.unique) val = ad.unique == UC_LO ? (long long)0x8000000000000000ull : 0x7fffffffffffffffll;  // (other aggregates read 0)
    } else {
      val = m.tmp1[s * 32 + lane];
    }
    const unsigned amask = m.act[s];
    if (amask == 0) continue;
    const bool active = (amask >> lane) & 1u;
    const uint32_t sl = m.slotv[s * 32 + lane];
    const uint32_t s0 = __shfl_sync(FULL, sl, __ffs(amask) - 1);
    const bool uni = __all_sync(FULL, !active || sl == s0);
    if (!uni) {
      if (cs != kNoSlot) {
        flush_agg(func, isf, cells + cs, part, lane);
        part = ident;
        cs = kNoSlot;
      }
      mixed_agg(func, isf, cells, sl, active, val, lane);
    } else {
      if (s0 != cs) {
        if (cs != kNoSlot) {
          flush_agg(func, isf, cells + cs, part, lane);
          part = ident;
        }
        cs = s0;
      }
      if (active) part = agg_combine(func, isf, part, val);
    }
  }
  m.acc[a * 32 + lane] = part;
}

// ---- fused fast path ---------------------------------------------------------------------------------------
// The dominant query shape runs in ONE pass over the vector with everything in registers:
//   filter  = conjunction of <= 2 range leaves on PLAIN non-null int64/double columns (or no filter)
//   keys    = <= 3 dictionary-string columns without NULLs in this row group, dense table
//   aggs    = counts + <= 2 Sum/Min/Max over PLAIN non-null columns read in place
// Eligibility of the QUERY is decided by the host (q.fast_ok).  Eligibility of the ROW GROUP (column
// kinds) is resolved once per row group into a FastPlan kept in the warp's shared memory; a row group
// that does not qualify sends its vectors down the general vectorized path.
constexpr int kFastLeaves = 2, kFastKeys = 3, kFastAggs = 2;
constexpr int kRgSmem = 2048;
constexpr uint32_t kVecChunk = 8;  // consecutive vectors a warp takes per turn  // row groups whose prefix table fits the CTA's shared memory

struct FastLeaf {
  uint32_t col_off;  // byte offset of the staged column inside a ring slot
  uint32_t flags;    // 1 compare as double, 2 column is double, 4 negate
  long long lo_i, hi_i;
  double lo_f, hi_f;
};
struct FastKey {
  const Run* runs;
  const uint8_t* stream;
  const uint32_t* lut;
  const Seed* seeds;    // global seeds of the row group
  int32_t seed_off;     // byte offset of the staged seed inside a ring slot, -1 = read the global one
  uint32_t stride;
};
struct FastAgg {
  uint32_t col_off;
  uint32_t func;  // AggFunc | is_float << 8
  int32_t index;  // index into q.aggs / q.t_agg
  uint32_t _pad;
};
struct IssueItem {
  const uint8_t* src;  // PLAIN: the chunk's value array; seed: the chunk's seed array
  uint32_t dst_off;    // byte offset inside a ring slot
  uint32_t is_seed;
};
struct IssuePlan {  // what to prefetch for a vector of the cached row group
  uint32_t n, _pad;
  IssueItem item[kMaxStagePlain + kMaxStageSeeds];
};
struct FastPlan {
  uint32_t ok, none, nl, nk, na, tight;
  FastLeaf leaf[kFastLeaves];
  FastKey key[kFastKeys];
  FastAgg agg[kFastAggs];
};

// lane 0 builds the plan of the warp's current row group from the cached descriptors
__device__ __noinline__ void build_fast_plan(const QueryDesc& q, const ChunkDesc* chunks, const LeafRt* lrt, FastPlan* fp) {
  fp->ok = 0;
  fp->none = 0;
  bool tight = true;
  uint32_t nl = 0, nk = 0, na = 0;
  for (int l = 0; l < q.n_leaves; l++) {
    const LeafDesc& ld = q.leaves[l];
    const uint8_t mode = lrt[l].mode;
    if (mode == LM_NONE) { fp->none = 1; continue; }
    if (mode == LM_ALL) continue;
    const ChunkDesc& c = chunks[ld.slot];
    const int p = q.slot_plain_stage[ld.slot];
    if (c.kind != CK_PLAIN64 || c.has_nulls || p < 0 || nl >= uint32_t(kFastLeaves)) return;
    FastLeaf& f = fp->leaf[nl++];
    f.col_off = uint32_t(p) * uint32_t(q.vl) * 8u;
    f.flags = (ld.cmp_float ? 1u : 0u) | (q.slot_type[ld.slot] == ST_F64 ? 2u : 0u) | (ld.neg ? 4u : 0u);
    f.lo_i = ld.lo_i; f.hi_i = ld.hi_i; f.lo_f = ld.lo_f; f.hi_f = ld.hi_f;
    if (f.flags != 0) tight = false;
  }
  for (int k = 0; k < q.n_keys; k++) {
    const KeyDesc& kd = q.keys[k];
    const ChunkDesc& c = chunks[kd.slot];
    if (c.kind == CK_ABSENT) continue;  // NULL for every row: contributes 0 to the dense slot
    if (c.kind != CK_DICT_STR || c.has_nulls || nk >= uint32_t(kFastKeys)) return;
    FastKey& f = fp->key[nk++];
    f.runs = c.runs; f.stream = c.values; f.lut = c.lut; f.seeds = c.seeds;
    const int sv = q.slot_seed_stage[kd.slot][0];
    f.seed_off = sv >= 0 ? int32_t(uint32_t(q.n_stage_plain) * uint32_t(q.vl) * 8u + uint32_t(sv) * uint32_t(sizeof(Seed))) : -1;
    f.stride = kd.dense_stride;
  }
  for (int a = 0; a < q.n_aggs; a++) {
    const AggDesc& ad = q.aggs[a];
    if (ad.func == 4) continue;
    const int slot = q.prog[ad.prog_off].slot;
    const ChunkDesc& c = chunks[slot];
    const int p = q.slot_plain_stage[slot];
    if (c.kind != CK_PLAIN64 || c.has_nulls || p < 0 || na >= uint32_t(kFastAggs)) return;
    FastAgg& f = fp->agg[na++];
    f.col_off = uint32_t(p) * uint32_t(q.vl) * 8u;
    f.func = uint32_t(ad.func) | (uint32_t(ad.is_float) << 8);
    f.index = a;
    if (f.func != 1u) tight = false;
  }
  fp->tight = tight ? 1u : 0u;
  fp->nl = nl; fp->nk = nk; fp->na = na;
  fp->ok = 1;
}

__device__ __noinline__ void build_issue_plan(const QueryDesc& q, const ChunkDesc* chunks, IssuePlan* ip) {
  uint32_t n = 0;
  for (int p = 0; p < q.n_stage_plain; p++) {
    const ChunkDesc& c = chunks[q.stage_plain_slot[p]];
    if (c.kind != CK_PLAIN64 || c.has_nulls) continue;
    ip->item[n].src = c.values;
    ip->item[n].dst_off = uint32_t(p) * uint32_t(q.vl) * 8u;
    ip->item[n].is_seed = 0;
    n++;
  }
  const uint32_t seed_base = uint32_t(q.n_stage_plain) * uint32_t(q.vl) * 8u;
  for (int t = 0; t < q.n_stage_seeds; t++) {
    const ChunkDesc& c = chunks[q.stage_seed_slot[t]];
    const bool is_def = q.stage_seed_is_def[t];
    const bool present = is_def ? (c.kind != CK_ABSENT && c.has_nulls) : (c.kind == CK_DICT_STR || c.kind == CK_DICT64);
    if (!present) continue;
    ip->item[n].src = reinterpret_cast<const uint8_t*>(is_def ? c.def_seeds : c.seeds);
    ip->item[n].dst_off = seed_base + uint32_t(t) * uint32_t(sizeof(Seed));
    ip->item[n].is_seed = 1;
    n++;
  }
  ip->n = n;
}

// Prefetch of a vector of the cached row group: everything resolved in the IssuePlan.
__device__ __forceinline__ void issue_cached(const QueryDesc& q, const IssuePlan& ip, uint32_t ring_saddr, uint32_t slot_bytes, int rs,
                                             uint32_t r0, uint32_t n_rows, int lane) {
  const uint32_t n = min(uint32_t(q.vl), n_rows - r0);
  const uint32_t plain_sz = (n * 8u + 15u) & ~15u;
  const uint32_t dst = ring_saddr + uint32_t(rs) * slot_bytes;
  for (uint32_t i = 0; i < ip.n; i++) {
    const IssueItem it = ip.item[i];
    if (it.is_seed) {
      if (lane < 2) cp_async16(dst + it.dst_off + uint32_t(lane) * 16u, it.src + size_t(r0 / kIndexRows) * sizeof(Seed) + lane * 16);
    } else {
      const uint8_t* src = it.src + size_t(r0) * 8 + uint32_t(lane) * 16u;
      const uint32_t d = dst + it.dst_off + uint32_t(lane) * 16u;
      if (n == uint32_t(q.vl)) {  // full vector: fixed trip count
        const uint32_t iters = uint32_t(q.vl) / 64u;
#pragma unroll 4
        for (uint32_t j = 0; j < iters; j++) cp_async16(d + j * 512u, src + j * 512u);
      } else {
        for (uint32_t o = uint32_t(lane) * 16u; o < plain_sz; o += 512u) cp_async16(d - uint32_t(lane) * 16u + o, src - uint32_t(lane) * 16u + o);
      }
    }
  }
  asm volatile("cp.async.commit_group;" ::: "memory");
}

__device__ __forceinline__ bool fast_leaf_test(const FastLeaf& f, long long x) {
  bool in;
  if (f.flags & 1u) {
    const double d = (f.flags & 2u) ? __longlong_as_double(x) : double(x);
    in = d >= f.lo_f && d <= f.hi_f;
  } else {
    in = x >= f.lo_i && x <= f.hi_i;
  }
  return in != ((f.flags & 4u) != 0);
}

// Slim run cursor of the fast path: the directory / stream / LUT pointers stay in the FastPlan.
struct KCur {
  uint32_t k, start, end, val, meta, off;
};
__device__ __forceinline__ void kc_advance(KCur& c, const FastKey& fk, uint32_t ord) {
  while (ord >= c.end) {
    c.k++;
    const uint4 r = __ldg(reinterpret_cast<const uint4*>(fk.runs + c.k));
    c.start = r.x; c.off = r.y; c.val = r.z; c.meta = r.w;
    c.end = __ldg(&fk.runs[c.k + 1].start);
  }
}
__device__ __forceinline__ uint32_t kc_get(KCur& c, const FastKey& fk, uint32_t ord) {
  if (ord >= c.end) kc_advance(c, fk, ord);
  if ((c.meta & 1u) == 0) return c.val;
  const uint32_t w = (c.meta >> 8) & 0xffu;
  return __ldg(fk.lut + extract_bits(fk.stream, c.off, uint64_t(ord - c.start) * w, w));
}

// Cold part of the fused pass: the step's active lanes are not all in the running group `cs`.
// Sorted parts produce exactly one shape here, a run boundary: the lanes still in `cs` join the running
// accumulators, the warp flushes once, and the remaining lanes (one new group) start the next run.
// Anything else (several new groups in one step) goes through the generic mixed path.
template <int NA>
__device__ __noinline__ void fast_cold_step(const QueryDesc& q, const FastPlan& fp, uint32_t slot, bool act, const long long (&val)[NA > 0 ? NA : 1],
                                            int lane, uint32_t& cs, uint32_t& cnt, long long (&part)[NA > 0 ? NA : 1]) {
  // 1. lanes that still belong to the running group
  if (cs != kNoSlot) {
    const bool old = act && slot == cs;
    if (__ballot_sync(FULL, act && !old) == 0) {  // (bit-packed boundary group that did not change the group)
      cnt += old ? 1u : 0u;
#pragma unroll
      for (int a = 0; a < NA; a++)
        if (old) part[a] = agg_combine(uint8_t(fp.agg[a].func & 0xff), (fp.agg[a].func >> 8) != 0, part[a], val[a]);
      return;
    }
    cnt += old ? 1u : 0u;
#pragma unroll
    for (int a = 0; a < NA; a++)
      if (old) part[a] = agg_combine(uint8_t(fp.agg[a].func & 0xff), (fp.agg[a].func >> 8) != 0, part[a], val[a]);
    act = act && !old;
    // 2. flush the running group
    const uint32_t tt = __reduce_add_sync(FULL, cnt);
    if (lane == 0 && tt) atomicAdd(q.t_rows + cs, (unsigned long long)tt);
    cnt = 0;
#pragma unroll
    for (int a = 0; a < NA; a++) {
      flush_agg(uint8_t(fp.agg[a].func & 0xff), (fp.agg[a].func >> 8) != 0, q.t_agg[fp.agg[a].index] + cs, part[a], lane);
      part[a] = agg_identity(uint8_t(fp.agg[a].func & 0xff), (fp.agg[a].func >> 8) != 0);
    }
    cs = kNoSlot;
  }
  // 3. what is left of the step
  const unsigned rest = __ballot_sync(FULL, act);
  if (rest == 0) return;
  const uint32_t s1 = __shfl_sync(FULL, slot, __ffs(rest) - 1);
  if (__all_sync(FULL, !act || slot == s1)) {  // one new group: it becomes the running group
    cs = s1;
    cnt = act ? 1u : 0u;
#pragma unroll
    for (int a = 0; a < NA; a++)
      if (act) part[a] = agg_combine(uint8_t(fp.agg[a].func & 0xff), (fp.agg[a].func >> 8) != 0, part[a], val[a]);
    return;
  }
  mixed_rows(q.t_rows, slot, act, lane);
#pragma unroll
  for (int a = 0; a < NA; a++)
    mixed_agg(uint8_t(fp.agg[a].func & 0xff), (fp.agg[a].func >> 8) != 0, q.t_agg[fp.agg[a].index], slot, act, val[a], lane);
}

template <int NL, int NK, int NA>
__device__ __noinline__ uint32_t fast_pass(const QueryDesc& q, uint8_t* wb, const FastPlan& fp, uint32_t slot_saddr,
                                            const uint8_t* slotmem, uint32_t r0, uint32_t chunk, uint32_t n_in, int steps, int lane,
                                            uint32_t cur_slot) {
  const WarpMem m = warp_mem(q, wb);
  // leaves: the active bound pair as raw 64-bit words
  long long llo[NL > 0 ? NL : 1], lhi[NL > 0 ? NL : 1];
  uint32_t lflags[NL > 0 ? NL : 1], lcol[NL > 0 ? NL : 1];
#pragma unroll
  for (int l = 0; l < NL; l++) {
    const FastLeaf& f = fp.leaf[l];
    lflags[l] = f.flags;
    lcol[l] = slot_saddr + f.col_off + uint32_t(lane) * 8u;
    llo[l] = (f.flags & 1u) ? __double_as_longlong(f.lo_f) : f.lo_i;
    lhi[l] = (f.flags & 1u) ? __double_as_longlong(f.hi_f) : f.hi_i;
  }
  KCur kc[NK > 0 ? NK : 1];
  uint32_t kstride[NK > 0 ? NK : 1];
#pragma unroll
  for (int k = 0; k < NK; k++) {
    const FastKey& fk = fp.key[k];
    const Seed* sd = fk.seed_off >= 0 ? reinterpret_cast<const Seed*>(slotmem + fk.seed_off) : fk.seeds + chunk;
    const uint4 a = *reinterpret_cast<const uint4*>(sd);
    const uint2 b = *(reinterpret_cast<const uint2*>(sd) + 2);
    kc[k].k = a.x; kc[k].start = a.y; kc[k].end = a.z; kc[k].off = a.w; kc[k].val = b.x; kc[k].meta = b.y;
    kstride[k] = fk.stride;
  }
  uint32_t acol[NA > 0 ? NA : 1];
  bool sum64[NA > 0 ? NA : 1];
  long long part[NA > 0 ? NA : 1];
#pragma unroll
  for (int a = 0; a < NA; a++) {
    acol[a] = slot_saddr + fp.agg[a].col_off + uint32_t(lane) * 8u;
    sum64[a] = fp.agg[a].func == 1u;  // Sum(int64): two adds in the hot loop
    part[a] = m.acc[fp.agg[a].index * 32 + lane];
  }
  uint32_t cs = cur_slot, cnt = m.cnt[lane], selected = 0;
  int s = 0;
  while (s < steps) {
    uint32_t slot = 0;
    bool act = false;
    // ---- hot loop: no calls inside, leaves only when the step is not entirely in the running group ----
#pragma unroll 1
    for (; s < steps; s++) {
      const uint32_t idx = uint32_t(s) * 32u + uint32_t(lane);
      act = idx < n_in;
#pragma unroll
      for (int l = 0; l < NL; l++) {
        const long long x = (long long)lds64(lcol[l] + uint32_t(s) * 256u);
        bool in;
        if (lflags[l] & 1u) {
          const double d = (lflags[l] & 2u) ? __longlong_as_double(x) : double(x);
          in = d >= __longlong_as_double(llo[l]) && d <= __longlong_as_double(lhi[l]);
        } else {
          in = x >= llo[l] && x <= lhi[l];
        }
        act = act && (in != ((lflags[l] & 4u) != 0));
      }
      const unsigned amask = __ballot_sync(FULL, act);
      if (amask == 0) continue;
      slot = 0;
      const uint32_t r = r0 + idx;
#pragma unroll
      for (int k = 0; k < NK; k++)
        if (act) slot += (kc_get(kc[k], fp.key[k], r) + 1u) * kstride[k];
      selected += __popc(amask);
      if (!__all_sync(FULL, !act || slot == cs)) break;  // group change: leave the hot loop
      cnt += act ? 1u : 0u;
#pragma unroll
      for (int a = 0; a < NA; a++) {
        const long long val = (long long)lds64(acol[a] + uint32_t(s) * 256u);
        if (sum64[a]) part[a] = (long long)((unsigned long long)part[a] + (act ? (unsigned long long)val : 0ull));
        else if (act) part[a] = agg_combine(uint8_t(fp.agg[a].func & 0xff), (fp.agg[a].func >> 8) != 0, part[a], val);
      }
    }
    if (s >= steps) break;
    // ---- cold: step s leaves the running group ----
    long long val[NA > 0 ? NA : 1];
#pragma unroll
    for (int a = 0; a < NA; a++) val[a] = (long long)lds64(acol[a] + uint32_t(s) * 256u);
    fast_cold_step<NA>(q, fp, slot, act, val, lane, cs, cnt, part);
    s++;
  }
  m.cnt[lane] = cnt;
#pragma unroll
  for (int a = 0; a < NA; a++) m.acc[fp.agg[a].index * 32 + lane] = part[a];
  if (lane == 0) m.selected[0] += selected;
  return cs;
}

// Tight variant of the fused pass, chosen per row group when every leaf is a plain (non-negated) int64
// range and every aggregate is Sum(int64).  The key cursors are WARP-UNIFORM: they sit on the runs that
// hold the first row of the current step, so the distance to the nearest run end says how many whole
// 32-row steps lie inside one group.  Those steps run in an inner loop with no vote, no shuffle and no
// branch (two loads, a range test, two adds).  A step that straddles one run end is split by lane index
// (lanes below the boundary close the running group, the others open the next one); only steps with a
// second boundary or a bit-packed run compute a slot per lane and go through fast_cold_step.
template <int NL, int NK, int NA>
__device__ __noinline__ uint32_t fast_pass_tight(const QueryDesc& q, uint8_t* wb, const FastPlan& fp, uint32_t slot_saddr,
                                                  const uint8_t* slotmem, uint32_t r0, uint32_t chunk, uint32_t n_in, int steps, int lane,
                                                  uint32_t cur_slot) {
  const WarpMem m = warp_mem(q, wb);
  long long lo[NL > 0 ? NL : 1], hi[NL > 0 ? NL : 1];
  uint32_t lcol[NL > 0 ? NL : 1];
#pragma unroll
  for (int l = 0; l < NL; l++) {
    lo[l] = fp.leaf[l].lo_i;
    hi[l] = fp.leaf[l].hi_i;
    lcol[l] = slot_saddr + fp.leaf[l].col_off + uint32_t(lane) * 8u;
  }
  uint32_t kk[NK > 0 ? NK : 1], kend[NK > 0 ? NK : 1], kadd[NK > 0 ? NK : 1];
  uint32_t kbp = 0;  // bit k: the current run of key k is bit-packed (kadd[k] is not valid)
#pragma unroll
  for (int k = 0; k < NK; k++) {
    const FastKey& fk = fp.key[k];
    const Seed* sd = fk.seed_off >= 0 ? reinterpret_cast<const Seed*>(slotmem + fk.seed_off) : fk.seeds + chunk;
    kk[k] = sd->k;
    kend[k] = sd->end;
    kadd[k] = (sd->val + 1u) * fk.stride;
    kbp |= (sd->meta & 1u) << k;
  }
  uint32_t acol[NA > 0 ? NA : 1];
  unsigned long long part[NA > 0 ? NA : 1];
#pragma unroll
  for (int a = 0; a < NA; a++) {
    acol[a] = slot_saddr + fp.agg[a].col_off + uint32_t(lane) * 8u;
    part[a] = (unsigned long long)m.acc[fp.agg[a].index * 32 + lane];
  }
  uint32_t cs = cur_slot, cnt = m.cnt[lane], sel = 0;
  const uint32_t rend = r0 + n_in;

  // moves the cursors onto the runs that hold `row` (same row in every lane: the loads broadcast)
  auto advance = [&](uint32_t row) {
#pragma unroll
    for (int k = 0; k < NK; k++) {
      if (row >= kend[k]) {
        const Run* runs = fp.key[k].runs;
        uint32_t i = kk[k], e;
        do {
          i++;
          e = __ldg(&runs[i + 1].start);
        } while (row >= e);
        kk[k] = i;
        kend[k] = e;
        const uint2 vm = __ldg(reinterpret_cast<const uint2*>(&runs[i].val));
        kadd[k] = (vm.x + 1u) * fp.key[k].stride;
        kbp = (kbp & ~(1u << k)) | ((vm.y & 1u) << k);
      }
    }
  };
  // the running group leaves the registers (Sum only: a group without rows has nothing to add)
  auto flush = [&]() {
    const uint32_t tt = __reduce_add_sync(FULL, cnt);
    if (tt == 0) return;
    if (lane == 0) atomicAdd(q.t_rows + cs, (unsigned long long)tt);
    cnt = 0;
#pragma unroll
    for (int a = 0; a < NA; a++) {
      unsigned long long v = part[a];
#pragma unroll
      for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(FULL, v, o);
      if (lane == 0) atomicAdd(reinterpret_cast<unsigned long long*>(q.t_agg[fp.agg[a].index] + cs), v);
      part[a] = 0;
    }
  };
  auto passes = [&](int s) -> bool {
    bool act = true;
#pragma unroll
    for (int l = 0; l < NL; l++) {
      const long long x = (long long)lds64(lcol[l] + uint32_t(s) * 256u);
      act = act && x >= lo[l] && x <= hi[l];
    }
    return act;
  };
  // slot of row r from the cursors (which sit on a row <= r); unpacks bit-packed runs
  auto lane_slot = [&](uint32_t r) -> uint32_t {
    uint32_t slot = 0;
#pragma unroll
    for (int k = 0; k < NK; k++) {
      const FastKey& fk = fp.key[k];
      uint32_t i = kk[k];
      while (r >= __ldg(&fk.runs[i + 1].start)) i++;
      const uint4 run = __ldg(reinterpret_cast<const uint4*>(fk.runs + i));
      uint32_t v = run.z;
      if (run.w & 1u) {
        const uint32_t w = (run.w >> 8) & 0xffu;
        v = __ldg(fk.lut + extract_bits(fk.stream, run.y, uint64_t(r - run.x) * w, w));
      }
      slot += (v + 1u) * fk.stride;
    }
    return slot;
  };
  auto general_step = [&](int s, uint32_t r, bool act) {
    const uint32_t slot = act ? lane_slot(r) : 0u;
    long long val[NA > 0 ? NA : 1], p2[NA > 0 ? NA : 1];
#pragma unroll
    for (int a = 0; a < NA; a++) {
      val[a] = (long long)lds64(acol[a] + uint32_t(s) * 256u);
      p2[a] = (long long)part[a];
    }
    fast_cold_step<NA>(q, fp, slot, act, val, lane, cs, cnt, p2);
#pragma unroll
    for (int a = 0; a < NA; a++) part[a] = (unsigned long long)p2[a];
  };

  int s = 0;
  while (s < steps) {
    uint32_t rs = r0 + uint32_t(s) * 32u;
    advance(rs);
    if (kbp != 0) {  // a long bit-packed run (unsorted key column): one slot per lane
      const uint32_t r = rs + uint32_t(lane);
      const bool act = r < rend && passes(s);
      sel += act ? 1u : 0u;
      general_step(s, r, act);
      s++;
      continue;
    }
    uint32_t safe = rend, us = 0;
#pragma unroll
    for (int k = 0; k < NK; k++) {
      safe = min(safe, kend[k]);
      us += kadd[k];
    }
    if (us != cs) {
      if (cs != kNoSlot) flush();
      cs = us;
    }
    // ---- whole steps inside the running group ----
    const int e = s + int((safe - rs) >> 5);
#pragma unroll 2
    for (; s < e; s++) {
      const bool act = passes(s);
      cnt += act ? 1u : 0u;
      sel += act ? 1u : 0u;
#pragma unroll
      for (int a = 0; a < NA; a++) part[a] += act ? lds64(acol[a] + uint32_t(s) * 256u) : 0ull;
    }
    if (s >= steps) break;
    // ---- the step that holds row `safe`: lanes below it still belong to the running group ----
    rs = r0 + uint32_t(s) * 32u;
    const uint32_t r = rs + uint32_t(lane);
    const bool act = r < rend && passes(s);
    const bool old = act && r < safe;
    sel += act ? 1u : 0u;
    cnt += old ? 1u : 0u;
#pragma unroll
    for (int a = 0; a < NA; a++) part[a] += old ? lds64(acol[a] + uint32_t(s) * 256u) : 0ull;
    if (safe < rend) {
      advance(safe);
      uint32_t safe2 = rend, us2 = 0;
#pragma unroll
      for (int k = 0; k < NK; k++) {
        safe2 = min(safe2, kend[k]);
        us2 += kadd[k];
      }
      const bool fresh = act && !old;
      if (kbp == 0 && safe2 >= min(rs + 32u, rend)) {  // one boundary in this step: the rest is one group
        if (us2 != cs) {
          flush();
          cs = us2;
        }
        cnt += fresh ? 1u : 0u;
#pragma unroll
        for (int a = 0; a < NA; a++) part[a] += fresh ? lds64(acol[a] + uint32_t(s) * 256u) : 0ull;
      } else {
        general_step(s, r, fresh);
      }
    }
    s++;
  }
  m.cnt[lane] = cnt;
#pragma unroll
  for (int a = 0; a < NA; a++) m.acc[fp.agg[a].index * 32 + lane] = (long long)part[a];
  sel = __reduce_add_sync(FULL, sel);
  if (lane == 0) m.selected[0] += sel;
  return cs;
}

template <int NL, int NK>
__device__ __forceinline__ uint32_t fast_dispatch_a(int na, const QueryDesc& q, uint8_t* m, const FastPlan& fp, uint32_t sa,
                                                    const uint8_t* sm, uint32_t r0, uint32_t chunk, uint32_t n_in, int steps, int lane,
                                                    uint32_t cs) {
  if (fp.tight) {
    switch (na) {
      case 0: return fast_pass_tight<NL, NK, 0>(q, m, fp, sa, sm, r0, chunk, n_in, steps, lane, cs);
      case 1: return fast_pass_tight<NL, NK, 1>(q, m, fp, sa, sm, r0, chunk, n_in, steps, lane, cs);
      default: return fast_pass_tight<NL, NK, 2>(q, m, fp, sa, sm, r0, chunk, n_in, steps, lane, cs);
    }
  }
  switch (na) {
    case 0: return fast_pass<NL, NK, 0>(q, m, fp, sa, sm, r0, chunk, n_in, steps, lane, cs);
    case 1: return fast_pass<NL, NK, 1>(q, m, fp, sa, sm, r0, chunk, n_in, steps, lane, cs);
    default: return fast_pass<NL, NK, 2>(q, m, fp, sa, sm, r0, chunk, n_in, steps, lane, cs);
  }
}
template <int NL>
__device__ __forceinline__ uint32_t fast_dispatch_k(int nk, int na, const QueryDesc& q, uint8_t* m, const FastPlan& fp, uint32_t sa,
                                                    const uint8_t* sm, uint32_t r0, uint32_t chunk, uint32_t n_in, int steps, int lane,
                                                    uint32_t cs) {
  switch (nk) {
    case 0: return fast_dispatch_a<NL, 0>(na, q, m, fp, sa, sm, r0, chunk, n_in, steps, lane, cs);
    case 1: return fast_dispatch_a<NL, 1>(na, q, m, fp, sa, sm, r0, chunk, n_in, steps, lane, cs);
    case 2: return fast_dispatch_a<NL, 2>(na, q, m, fp, sa, sm, r0, chunk, n_in, steps, lane, cs);
    default: return fast_dispatch_a<NL, 3>(na, q, m, fp, sa, sm, r0, chunk, n_in, steps, lane, cs);
  }
}
__device__ __forceinline__ uint32_t fast_dispatch(const VecCtx& v, uint8_t* m, const FastPlan& fp, int lane, uint32_t cs) {
  const QueryDesc& q = *v.q;
  const uint32_t sa = smem_u32(v.slotmem);
  const uint32_t n_in = min(uint32_t(q.vl), v.n_rows - v.r0);
  switch (fp.nl) {
    case 0: return fast_dispatch_k<0>(int(fp.nk), int(fp.na), q, m, fp, sa, v.slotmem, v.r0, v.chunk, n_in, v.steps, lane, cs);
    case 1: return fast_dispatch_k<1>(int(fp.nk), int(fp.na), q, m, fp, sa, v.slotmem, v.r0, v.chunk, n_in, v.steps, lane, cs);
    default: return fast_dispatch_k<2>(int(fp.nk), int(fp.na), q, m, fp, sa, v.slotmem, v.r0, v.chunk, n_in, v.steps, lane, cs);
  }
}

__global__ void __launch_bounds__(kVecThreads, 4) k_scan(const QueryDesc* __restrict__ qp) {
  extern __shared__ __align__(128) uint8_t dyn[];
  __shared__ QueryDesc sq;
  {
    const uint32_t* src = reinterpret_cast<const uint32_t*>(qp);
    uint32_t* dst = reinterpret_cast<uint32_t*>(&sq);
    for (uint32_t i = threadIdx.x; i < sizeof(QueryDesc) / 4; i += blockDim.x) dst[i] = src[i];
  }
  __syncthreads();
  const QueryDesc& q = sq;
  const bool rg_in_smem = q.n_rg <= kRgSmem;
  uint32_t* const s_first = reinterpret_cast<uint32_t*>(dyn + size_t(blockDim.x >> 5) * q.wr_bytes);  // after the warp regions
  if (rg_in_smem)
    for (int i = threadIdx.x; i <= q.n_rg; i += blockDim.x) s_first[i] = __ldg(&q.rg_first_tile[i]);
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint8_t* const wb = dyn + size_t(warp) * q.wr_bytes;  // this warp's shared-memory region (see WarpMem)
  const int D = q.n_ring;
  uint32_t cached_rows = 0;
  if (lane == 0) reinterpret_cast<unsigned long long*>(wb + q.wr_acc + size_t(q.n_aggs) * 32 * 8)[0] = 0;
  reinterpret_cast<uint32_t*>(wb + q.wr_acc + size_t(q.n_aggs) * 32 * 8 + 16)[lane] = 0;
  reinterpret_cast<uint32_t*>(wb + q.wr_acc + size_t(q.n_aggs) * 32 * 8 + 16 + 32 * 4)[lane] = kNoSlot;
  for (int a = 0; a < q.n_aggs; a++) reinterpret_cast<long long*>(wb + q.wr_acc)[a * 32 + lane] = agg_identity(q.aggs[a].func, q.aggs[a].is_float);
  __syncwarp();

  const uint32_t gw = blockIdx.x * (blockDim.x >> 5) + warp;  // global warp id
  const uint32_t GW = gridDim.x * (blockDim.x >> 5);
  const bool dense = q.table_mode == TM_DENSE;
  uint32_t cur_slot = kNoSlot;  // warp-uniform running group
  bool overflow = false;

  // Row-group lookup without pointer chasing: the prefix table sits in shared memory and every warp
  // walks it monotonically (its vectors only move forward); the descriptors of the row group a warp
  // is in are cached in the warp's shared-memory region, together with the resolved fast-path and
  // prefetch plans.  Vectors are dealt in chunks of kVecChunk consecutive vectors (warp g takes chunks
  // g, g + GW, ...), so a warp stays in one row group for a whole chunk while selective filters still
  // spread evenly over the warps.
  auto first_tile = [&](int i) -> uint32_t { return rg_in_smem ? s_first[i] : __ldg(&q.rg_first_tile[i]); };
  auto nth_vec = [&](uint32_t i) -> uint32_t { return ((i / kVecChunk) * GW + gw) * kVecChunk + (i % kVecChunk); };
  int rg = 0, rg_a = 0;          // row group of the vector being processed / being prefetched
  int cached_rg = -1;
  const uint32_t ring_saddr = smem_u32(wb + q.wr_ring);
  IssuePlan* const iplan = reinterpret_cast<IssuePlan*>(wb + q.wr_iplan);
  auto issue = [&](uint32_t vec, int rs) {
    if (vec >= q.n_tiles) {
      asm volatile("cp.async.commit_group;" ::: "memory");
      return;
    }
    while (vec >= first_tile(rg_a + 1)) rg_a++;
    if (rg_a == cached_rg)
      issue_cached(q, *iplan, ring_saddr, q.slot_bytes, rs, (vec - first_tile(rg_a)) * q.vl, cached_rows, lane);
    else
      issue_vector(q, wb + q.wr_ring, vec, rs, first_tile(rg_a), __ldg(&q.rg_rows[rg_a]), q.chunks + size_t(rg_a) * q.n_slots, lane);
  };

  // prologue: fill the ring (every iteration commits exactly one cp.async group, empty ones included,
  // so that "at most D-1 groups pending" always means "the current vector has landed")
  for (int d = 0; d < D - 1; d++) issue(nth_vec(uint32_t(d)), d);
  int rs = 0, rs_ahead = D - 1;
  for (uint32_t it = 0;; it++) {
    const uint32_t vec = nth_vec(it);
    if (vec >= q.n_tiles) break;
    while (vec >= first_tile(rg + 1)) rg++;
    if (rg != cached_rg) {  // warp-uniform: copy this row group's descriptors into shared memory
      const uint32_t* src = reinterpret_cast<const uint32_t*>(q.chunks + size_t(rg) * q.n_slots);
      uint32_t* dst = reinterpret_cast<uint32_t*>(reinterpret_cast<ChunkDesc*>(wb + q.wr_cdesc));
      for (uint32_t i = lane; i < uint32_t(q.n_slots) * sizeof(ChunkDesc) / 4; i += 32) dst[i] = __ldg(src + i);
      src = reinterpret_cast<const uint32_t*>(q.leaf_rt + size_t(rg) * q.n_leaves);
      dst = reinterpret_cast<uint32_t*>(reinterpret_cast<LeafRt*>(wb + q.wr_clrt));
      for (uint32_t i = lane; i < uint32_t(q.n_leaves) * sizeof(LeafRt) / 4; i += 32) dst[i] = __ldg(src + i);
      if (q.bool_keys) load_bool_keys(q, wb, rg, cached_rg < 0, lane);
      cached_rg = rg;
      cached_rows = __ldg(&q.rg_rows[rg]);
      __syncwarp();
      if (lane == 0) {
        build_issue_plan(q, reinterpret_cast<ChunkDesc*>(wb + q.wr_cdesc), iplan);
        if (q.fast_ok)
          build_fast_plan(q, reinterpret_cast<ChunkDesc*>(wb + q.wr_cdesc), reinterpret_cast<LeafRt*>(wb + q.wr_clrt), reinterpret_cast<FastPlan*>(wb + q.wr_fplan));
      }
      __syncwarp();
    }
    issue(nth_vec(it + uint32_t(D) - 1), rs_ahead);
    rs_ahead = (rs_ahead + 1 == D) ? 0 : rs_ahead + 1;
    VecCtx v;
    v.q = &q;
    v.n_rows = cached_rows;
    v.r0 = (vec - first_tile(rg)) * q.vl;
    v.chunk = v.r0 / kIndexRows;
    v.chunks = reinterpret_cast<ChunkDesc*>(wb + q.wr_cdesc);
    v.lrt = reinterpret_cast<LeafRt*>(wb + q.wr_clrt);
    v.slotmem = (wb + q.wr_ring) + size_t(rs) * q.slot_bytes;
    v.steps = int((min(uint32_t(q.vl), v.n_rows - v.r0) + 31) / 32);
    // the vector's copies are the oldest pending group of every lane
    if (D == 2) cp_async_wait<1>();
    else if (D == 3) cp_async_wait<2>();
    else cp_async_wait<3>();
    __syncwarp();

    if (q.fast_ok && reinterpret_cast<FastPlan*>(wb + q.wr_fplan)->ok) {
      if (!reinterpret_cast<FastPlan*>(wb + q.wr_fplan)->none) cur_slot = fast_dispatch(v, wb, *reinterpret_cast<FastPlan*>(wb + q.wr_fplan), lane, cur_slot);  // one fused pass
    } else if (vec_selection(v, wb, lane) != 0) {
      if (dense) vec_slots_dense(v, wb, lane);
      else overflow |= vec_slots_hash(v, wb, lane);
      const uint32_t end_slot = vec_count_rows(v, wb, lane, cur_slot);
      for (int a = 0; a < q.n_aggs; a++)
        if (q.aggs[a].func != 4 /*count*/) vec_aggregate(v, wb, a, lane, cur_slot);
      cur_slot = end_slot;
    }
    __syncwarp();  // every lane is done with ring slot rs before it is refilled
    rs = (rs + 1 == D) ? 0 : rs + 1;
  }
  // ---- final flush ---------------------------------------------------------------------------------
  if (cur_slot != kNoSlot) {
    const uint32_t tt = __reduce_add_sync(FULL, reinterpret_cast<uint32_t*>(wb + q.wr_acc + size_t(q.n_aggs) * 32 * 8 + 16)[lane]);
    if (lane == 0 && tt) atomicAdd(q.t_rows + cur_slot, (unsigned long long)tt);
    for (int a = 0; a < q.n_aggs; a++) {
      if (q.aggs[a].func == 4) continue;
      flush_agg(q.aggs[a].func, q.aggs[a].is_float, q.t_agg[a] + cur_slot, reinterpret_cast<long long*>(wb + q.wr_acc)[a * 32 + lane], lane);
    }
  }
  if (lane == 0 && reinterpret_cast<unsigned long long*>(wb + q.wr_acc + size_t(q.n_aggs) * 32 * 8)[0]) atomicAdd(q.counters + 0, reinterpret_cast<unsigned long long*>(wb + q.wr_acc + size_t(q.n_aggs) * 32 * 8)[0]);
  if (overflow) atomicExch(q.counters + 1, 1ull);
}

// ======================================================================================================
// k_rows: predicate + order-preserving compaction of the projected columns
// ======================================================================================================
// Selected rows of the warp's 128-row chunk: bit j = this lane's row of step j passes the predicate.  Every slot a
// leaf reads is decoded once for all of its leaves into leafbits[j] (bit l = leaf l selects row j).
// NULL semantics: binaryscalarexpr.go:143-150 (numeric NULL never selected), :165-172,:205-212
// (dictionary == NULL / != NULL), missing columns :47-73 (LM_ALL / LM_NONE precomputed on the host).
__device__ __forceinline__ uint32_t chunk_selection(const QueryDesc& q, const ChunkDesc* chunks, const LeafRt* __restrict__ lrt,
                                                    uint32_t chunk, uint32_t n_rows, int lane) {
  const uint32_t c0 = chunk * kIndexRows;
  uint32_t actbits = 0;
  if (q.n_filter_prog == 0) {
#pragma unroll
    for (int j = 0; j < STEPS; j++)
      if (c0 + j * 32 + lane < n_rows) actbits |= 1u << j;
    return actbits;
  }
  uint32_t cbits = 0;
  for (int l = 0; l < q.n_leaves; l++)
    if (lrt[l].mode == LM_ALL) cbits |= 1u << l;
  uint32_t leafbits[STEPS];
#pragma unroll
  for (int j = 0; j < STEPS; j++) leafbits[j] = cbits;
  for (int slot = 0; slot < q.n_slots; slot++) {
    if (!q.slot_used_by_leaf[slot]) continue;
    if (q.slot_type[slot] == ST_DICT) {
      DictReader rd;
      rd.init(chunks[slot], chunk, lane);
      uint32_t gid[STEPS];
#pragma unroll
      for (int j = 0; j < STEPS; j++) gid[j] = rd.next(c0 + j * 32 + lane, n_rows);
      for (int l = 0; l < q.n_leaves; l++) {
        if (q.leaves[l].slot != slot || lrt[l].mode != LM_EVAL) continue;
        const uint8_t* lut = lrt[l].lut;
        const uint32_t nullres = lrt[l].null_result;
#pragma unroll
        for (int j = 0; j < STEPS; j++) {
          uint32_t r = (gid[j] == kNullIdx) ? nullres : uint32_t(__ldg(lut + gid[j]));
          leafbits[j] |= (r & 1u) << l;
        }
      }
    } else {
      NumReader rd;
      rd.init(chunks[slot], chunk, lane);
      long long bits[STEPS];
      bool null[STEPS];
#pragma unroll
      for (int j = 0; j < STEPS; j++) bits[j] = rd.next(c0 + j * 32 + lane, n_rows, null[j]);
      const bool f64col = q.slot_type[slot] == ST_F64;
      for (int l = 0; l < q.n_leaves; l++) {
        const LeafDesc& ld = q.leaves[l];
        if (ld.slot != slot || lrt[l].mode != LM_EVAL) continue;
#pragma unroll
        for (int j = 0; j < STEPS; j++) leafbits[j] |= uint32_t(!null[j] && leaf_range(ld, bits[j], f64col)) << l;
      }
    }
  }
#pragma unroll
  for (int j = 0; j < STEPS; j++)
    if (c0 + j * 32 + lane < n_rows && eval_filter(q, leafbits[j])) actbits |= 1u << j;
  return actbits;
}

// At least two CTAs per SM: without a minimum, ptxas spills registers to fit four.
__global__ void __launch_bounds__(NT, 2) k_rows(const QueryDesc* __restrict__ qp) {
  __shared__ QueryDesc sq;
  __shared__ uint32_t warp_cnt[NWARP];
  __shared__ unsigned long long tile_base_s;
  __shared__ uint32_t tile_ticket;
  {
    const uint32_t* src = reinterpret_cast<const uint32_t*>(qp);
    uint32_t* dst = reinterpret_cast<uint32_t*>(&sq);
    for (uint32_t i = threadIdx.x; i < sizeof(QueryDesc) / 4; i += NT) dst[i] = src[i];
  }
  __syncthreads();
  const QueryDesc& q = sq;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t lt = (1u << lane) - 1u;
  volatile unsigned long long* state = q.tile_state;  // [n_tiles]: bits 62..63 flag (1 aggregate, 2 prefix), low bits value

  for (;;) {
    // tiles are handed out in order so that every predecessor of a tile is running or finished
    if (threadIdx.x == 0) tile_ticket = atomicAdd(reinterpret_cast<unsigned int*>(q.counters + 2), 1u);
    __syncthreads();
    const uint32_t tile = tile_ticket;
    if (tile >= q.n_tiles) break;
    const int rg = find_rg(q.rg_first_tile, q.n_rg, tile);
    const uint32_t tile_in_rg = tile - __ldg(&q.rg_first_tile[rg]);
    const uint32_t n_rows = __ldg(&q.rg_rows[rg]);
    const uint32_t chunk = tile_in_rg * NWARP + warp, c0 = chunk * kIndexRows;
    const ChunkDesc* chunks = q.chunks + size_t(rg) * q.n_slots;

    uint32_t actbits = 0;
    if (c0 < n_rows) actbits = chunk_selection(q, chunks, q.leaf_rt + size_t(rg) * q.n_leaves, chunk, n_rows, lane);
    // rank of every selected row inside the warp's chunk, in row order
    uint32_t rank[STEPS];
    uint32_t wtotal = 0;
#pragma unroll
    for (int j = 0; j < STEPS; j++) {
      unsigned m = __ballot_sync(FULL, (actbits >> j) & 1u);
      rank[j] = wtotal + __popc(m & lt);
      wtotal += __popc(m);
    }
    if (lane == 0) warp_cnt[warp] = wtotal;
    __syncthreads();
    uint32_t wbase = 0, ttotal = 0;
    for (int w = 0; w < NWARP; w++) {
      if (w < warp) wbase += warp_cnt[w];
      ttotal += warp_cnt[w];
    }
    // decoupled look-back over the preceding tiles (one warp, 32 predecessors per probe)
    if (warp == 0) {
      if (lane == 0) state[tile] = (1ull << 62) | ttotal;
      __threadfence();
      unsigned long long excl = 0;
      int64_t look = int64_t(tile) - 1;
      while (look >= 0) {
        int64_t tt = look - lane;
        unsigned long long s = (tt >= 0) ? state[tt] : (2ull << 62);
        while (__any_sync(FULL, (s >> 62) == 0)) s = (tt >= 0) ? state[tt] : (2ull << 62);  // predecessors publish soon
        unsigned pmask = __ballot_sync(FULL, (s >> 62) == 2);
        int first_prefix = pmask ? __ffs(pmask) - 1 : 32;
        unsigned long long contrib = (lane <= first_prefix) ? (s & ((1ull << 62) - 1)) : 0;
        contrib = warp_reduce(contrib, [](unsigned long long a, unsigned long long b) { return a + b; });
        excl += contrib;
        if (pmask) break;
        look -= 32;
      }
      if (lane == 0) {
        __threadfence();
        state[tile] = (2ull << 62) | (excl + ttotal);
        tile_base_s = excl;
      }
    }
    __syncthreads();
    const unsigned long long base = tile_base_s + wbase;
    // ---- write the projected columns of the selected rows ---------------------------------------
    if (c0 < n_rows && wtotal > 0) {
      for (int o = 0; o < q.n_out; o++) {
        const int slot = q.out_slot[o];
        if (q.slot_type[slot] == ST_DICT) {
          DictReader rd;
          rd.init(chunks[slot], chunk, lane);
          int32_t* out = reinterpret_cast<int32_t*>(q.out_data[o]);
#pragma unroll
          for (int j = 0; j < STEPS; j++) {
            const uint32_t gid = rd.next(c0 + j * 32 + lane, n_rows);
            if ((actbits >> j) & 1u) out[base + rank[j]] = (gid == kNullIdx) ? -1 : int32_t(gid);
          }
        } else {
          NumReader rd;
          rd.init(chunks[slot], chunk, lane);
          long long* out = reinterpret_cast<long long*>(q.out_data[o]);
          uint8_t* valid = q.out_valid[o];
#pragma unroll
          for (int j = 0; j < STEPS; j++) {
            bool null;
            const long long v = rd.next(c0 + j * 32 + lane, n_rows, null);
            if ((actbits >> j) & 1u) {
              out[base + rank[j]] = v;
              valid[base + rank[j]] = null ? 0 : 1;
            }
          }
        }
      }
    }
    if (threadIdx.x == 0 && tile + 1 == q.n_tiles) q.counters[0] = tile_base_s + ttotal;  // total selected rows
    __syncthreads();
  }
}

// ======================================================================================================
// k_table_init: rows = 0, sum = 0, min = +max, max = -max (int64) / +-inf (double), tags = 0
// ======================================================================================================
__global__ void k_table_init(QueryDesc q, bool zero_counters) {
  if (zero_counters && blockIdx.x == 0 && threadIdx.x < 10) q.counters[threadIdx.x] = 0;  // counters + the group counter behind them
  const size_t stride = size_t(gridDim.x) * blockDim.x;
  for (size_t s = size_t(blockIdx.x) * blockDim.x + threadIdx.x; s < q.table_slots; s += stride) {
    q.t_rows[s] = 0;
    if (q.table_mode == TM_HASH) q.t_tag[s] = 0;
    for (int a = 0; a < q.n_aggs; a++) {
      const AggDesc& ad = q.aggs[a];
      if (ad.func != 4) q.t_agg[a][s] = agg_identity(ad.func, ad.is_float);
    }
  }
}

// ======================================================================================================
// k_finalize
// ======================================================================================================
__global__ void k_finalize(FinalizeDesc f) {
  const size_t stride = size_t(gridDim.x) * blockDim.x;
  for (size_t s = size_t(blockIdx.x) * blockDim.x + threadIdx.x; s < f.table_slots; s += stride) {
    unsigned long long rows = f.t_rows[s];
    if (rows == 0) continue;
    unsigned int o = atomicAdd(f.out_count, 1u);
    if (o >= f.max_out) continue;
    f.out_rows[o] = rows;
    for (int k = 0; k < f.n_keys; k++) {
      const KeyDesc& kd = f.keys[k];
      long long code;
      if (f.table_mode == TM_DENSE) {
        code = (long long)((s / kd.dense_stride) % f.dense_radix[k]);
      } else {
        unsigned long long w = f.t_keys[s * f.key_words + kd.word];
        if (kd.is_int64) code = (long long)w;
        else code = (long long)((w >> kd.shift) & ((kd.bits >= 64) ? ~0ull : ((1ull << kd.bits) - 1ull)));
      }
      f.out_keys[size_t(k) * f.max_out + o] = code;
    }
    for (int a = 0; a < f.n_aggs; a++) {
      const long long v = f.t_agg[a] ? f.t_agg[a][s] : (long long)rows;
      if (f.agg_unique[a] == UC_HI) {  // Unique: the value where both cells meet, else NULL (0); this column: validity bytes
        const long long lo = f.t_agg[a - 1][s];
        f.out_aggs[size_t(a - 1) * f.max_out + o] = lo == v ? lo : 0;
        reinterpret_cast<uint8_t*>(f.out_aggs + size_t(a) * f.max_out)[o] = lo == v;
      } else {
        f.out_aggs[size_t(a) * f.max_out + o] = v;
      }
    }
  }
}

// ======================================================================================================
// k_merge: fold one remote partial table (same QueryDesc shape, S source slots) into the local one.  Hash-mode
// tables of different ranks may differ in S (each rank sizes its table from its own rows); a dense table has the
// local table's S.
// Partial layout (position independent): [rows u64 x S][stored agg i64 x S]...[tags u32 x S (8-aligned)][keys u64 x S*W]
// ======================================================================================================
__global__ void k_merge(QueryDesc q, const uint8_t* __restrict__ partial, size_t S) {
  const unsigned long long* p_rows = reinterpret_cast<const unsigned long long*>(partial);
  const long long* p_agg = reinterpret_cast<const long long*>(partial + S * 8);
  int n_stored = 0;
  int agg_pos[kMaxAggs];
  for (int a = 0; a < q.n_aggs; a++) agg_pos[a] = (q.aggs[a].func == 4) ? -1 : n_stored++;
  const unsigned long long* p_keys =
      reinterpret_cast<const unsigned long long*>(partial + S * 8 * (1 + n_stored) + ((S * 4 + 7) & ~size_t(7)));
  bool overflow = false;
  const size_t stride = size_t(gridDim.x) * blockDim.x;
  for (size_t s = size_t(blockIdx.x) * blockDim.x + threadIdx.x; s < S; s += stride) {
    unsigned long long rows = p_rows[s];
    if (rows == 0) continue;
    uint32_t dst;
    if (q.table_mode == TM_DENSE) {
      dst = uint32_t(s);
    } else {
      unsigned long long kw[kMaxKeyWords];
      for (int w = 0; w < kMaxKeyWords; w++) kw[w] = (w < q.key_words) ? p_keys[s * q.key_words + w] : 0;
      dst = hash_find_or_insert<kMaxKeyWords>(q, kw, &overflow);
      if (overflow) break;
    }
    atomicAdd(q.t_rows + dst, rows);
    for (int a = 0; a < q.n_aggs; a++) {
      if (agg_pos[a] < 0) continue;
      apply_agg(q.aggs[a].func, q.aggs[a].is_float, q.t_agg[a] + dst, p_agg[size_t(agg_pos[a]) * S + s]);
    }
  }
  if (overflow) atomicExch(q.counters + 1, 1ull);
}

// ======================================================================================================
// k_decode: one column chunk -> dense buffers (K1 standalone).
//   DICT_STR : out_i32[row] = global dictionary id, -1 for NULL
//   numeric  : out_i64[row] = value (0 for NULL), out_valid[row] = 0/1
// ======================================================================================================
__global__ void __launch_bounds__(NT) k_decode(ChunkDesc c, uint32_t n_chunks, int32_t* __restrict__ out_i32,
                                               long long* __restrict__ out_i64, uint8_t* __restrict__ out_valid) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (uint32_t chunk = blockIdx.x * NWARP + warp; chunk < n_chunks; chunk += gridDim.x * NWARP) {
    const uint32_t c0 = chunk * kIndexRows;
    if (c.kind == CK_DICT_STR) {
      DictReader rd;
      rd.init(c, chunk, lane);
      uint32_t gid[STEPS];
#pragma unroll
      for (int j = 0; j < STEPS; j++) gid[j] = rd.next(c0 + j * 32 + lane, c.n_rows);
#pragma unroll
      for (int j = 0; j < STEPS; j++) {
        const uint32_t r = c0 + j * 32 + lane;
        if (r < c.n_rows) out_i32[r] = (gid[j] == kNullIdx) ? -1 : int32_t(gid[j]);
      }
    } else {
      NumReader rd;
      rd.init(c, chunk, lane);
      long long v[STEPS];
      bool null[STEPS];
#pragma unroll
      for (int j = 0; j < STEPS; j++) v[j] = rd.next(c0 + j * 32 + lane, c.n_rows, null[j]);
#pragma unroll
      for (int j = 0; j < STEPS; j++) {
        const uint32_t r = c0 + j * 32 + lane;
        if (r < c.n_rows) {
          out_i64[r] = v[j];
          out_valid[r] = null[j] ? 0 : 1;
        }
      }
    }
  }
}

// ======================================================================================================
// host launchers
// ======================================================================================================
namespace {
struct KernelConfig {
  size_t smem_limit = 0;                       // dynamic shared memory limit raised so far (0: the default)
  std::map<std::pair<int, size_t>, int> ctas;  // (threads, dynamic shared memory) -> resident CTAs per SM
};
std::mutex config_mu;
std::map<std::pair<int, const void*>, KernelConfig> configs;  // (device, kernel), guarded by config_mu

cudaError_t kernel_config(const void* kern, KernelConfig** out) {  // (config_mu held)
  int dev = 0;
  const cudaError_t e = cudaGetDevice(&dev);
  if (e == cudaSuccess) *out = &configs[{dev, kern}];
  return e;
}

int grid_for(size_t n) {
  int blocks = int((n + 255) / 256);
  if (blocks > 132 * 8) blocks = 132 * 8;  // 8 CTAs per SM of an H100 SXM (132 SMs), grid-stride beyond
  return blocks < 1 ? 1 : blocks;
}
}  // namespace

cudaError_t kernel_smem_at_least(const void* kern, size_t smem) {
  std::lock_guard<std::mutex> lock(config_mu);
  KernelConfig* k = nullptr;
  cudaError_t e = kernel_config(kern, &k);
  if (e != cudaSuccess || smem <= k->smem_limit) return e;
  e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem));
  if (e == cudaSuccess) k->smem_limit = smem;
  return e;
}

cudaError_t kernel_ctas_per_sm(const void* kern, int threads, size_t smem, int* per_sm) {
  std::lock_guard<std::mutex> lock(config_mu);
  KernelConfig* k = nullptr;
  cudaError_t e = kernel_config(kern, &k);
  if (e != cudaSuccess) return e;
  auto it = k->ctas.find({threads, smem});
  if (it == k->ctas.end()) {
    int n = 0;
    e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, kern, threads, smem);
    if (e != cudaSuccess) return e;
    it = k->ctas.emplace(std::make_pair(threads, smem), std::max(n, 1)).first;
  }
  *per_sm = it->second;
  return cudaSuccess;
}

cudaError_t launch_table_init(const QueryDesc& q, cudaStream_t st, bool zero_counters) {
  k_table_init<<<grid_for(q.table_slots), 256, 0, st>>>(q, zero_counters);
  return cudaGetLastError();
}

cudaError_t launch_scan(const QueryDesc* d_q, const QueryDesc& q, int sm_count, cudaStream_t st) {
  if (q.n_tiles == 0) return cudaSuccess;
  const int warps = kVecThreads / 32;
  const size_t smem = size_t(q.wr_bytes) * warps + (q.n_rg <= 2048 ? (size_t(q.n_rg) + 1) * 4 + 16 : 0);
  const void* kern = reinterpret_cast<const void*>(k_scan);
  int per_sm = 0;
  cudaError_t e = kernel_smem_at_least(kern, smem);
  if (e == cudaSuccess) e = kernel_ctas_per_sm(kern, kVecThreads, smem, &per_sm);
  if (e != cudaSuccess) return e;
  uint32_t grid = uint32_t(sm_count) * uint32_t(per_sm);
  const uint32_t need = (q.n_tiles + warps - 1) / warps;
  if (grid > need) grid = need;
  k_scan<<<grid, kVecThreads, smem, st>>>(d_q);
  return cudaGetLastError();
}

cudaError_t launch_rows(const QueryDesc* d_q, const QueryDesc& q, int sm_count, cudaStream_t st) {
  if (q.n_tiles == 0) return cudaSuccess;
  int per_sm = 0;
  cudaError_t e = kernel_ctas_per_sm(reinterpret_cast<const void*>(k_rows), NT, 0, &per_sm);
  if (e != cudaSuccess) return e;
  uint32_t grid = uint32_t(sm_count) * uint32_t(per_sm);
  if (grid > q.n_tiles) grid = q.n_tiles;
  k_rows<<<grid, NT, 0, st>>>(d_q);
  return cudaGetLastError();
}

cudaError_t launch_finalize(const FinalizeDesc& f, cudaStream_t st) {
  k_finalize<<<grid_for(f.table_slots), 256, 0, st>>>(f);
  return cudaGetLastError();
}

// ======================================================================================================
// k_finalize_dense: occupied slots of a dense table -> compacted columns (one warp-aggregated atomic per warp)
// ======================================================================================================
__global__ void __launch_bounds__(256) k_finalize_dense(DenseOut f) {
  // f.hdr: 256-byte header in DEVICE memory (zero on entry, left zero on exit): [0] rows written, [16 + k] key k has a
  // NULL, [62] CTAs done.  f.out may be page-locked HOST memory (the columns then cross PCIe as they are produced and
  // no copy operation follows the kernel).  The last CTA to finish publishes the header in front of the columns and
  // clears the working copy, so no memset precedes the next launch.
  uint32_t* hdr = f.hdr;
  const size_t key_bytes = (size_t(f.max_out) * 4 + 7) & ~size_t(7);
  const int lane = threadIdx.x & 31;
  const size_t stride = size_t(gridDim.x) * blockDim.x;
  const size_t S = f.table_slots, S_pad = (S + 31) & ~size_t(31);
  bool failed = false;
  if (f.n_src > 0) {
    // collective Execute: every CTA waits for the peers' flags itself (they are written into this rank's own memory)
    __shared__ int bad;
    if (threadIdx.x == 0) bad = 0;
    __syncthreads();
    if (int(threadIdx.x) < f.n_src) {
      const int r = threadIdx.x;
      unsigned long long t0 = 0, seen;
      unsigned spins = 0;
      for (;;) {
        asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(seen) : "l"(f.flags + 2 * r) : "memory");
        if (seen >= f.seq) break;
        __nanosleep(100);
        if ((++spins & 1023u) == 0) {
          unsigned long long now;
          asm volatile("mov.u64 %0, %globaltimer;" : "=l"(now));
          if (t0 == 0) t0 = now;
          else if (now - t0 > f.timeout_ns) { atomicExch(&bad, 1); break; }
        }
      }
      if (seen >= f.seq && f.flags[2 * r + 1] != f.bytes) atomicExch(&bad, 2);
    }
    __syncthreads();
    __threadfence();
    if (bad) {
      failed = true;
      if (threadIdx.x == 0) atomicExch(f.err, (unsigned long long)bad);
    }
  }
  for (size_t s = size_t(blockIdx.x) * blockDim.x + threadIdx.x; s < S_pad && !failed; s += stride) {
    unsigned long long rows = 0;
    if (s < S) {
      if (f.n_src > 0) {
        for (int r = 0; r < f.n_src; r++) rows += reinterpret_cast<const unsigned long long*>(f.src[r])[s];
      } else {
        rows = f.t_rows[s];
      }
    }
    const unsigned m = __ballot_sync(FULL, rows != 0);
    if (m == 0) continue;
    uint32_t base = 0;
    if (lane == 0) base = atomicAdd(hdr, uint32_t(__popc(m)));
    base = __shfl_sync(FULL, base, 0);
    if (rows == 0) continue;
    const uint32_t o = base + __popc(m & ((1u << lane) - 1u));
    if (o >= f.max_out) continue;
    for (uint32_t k = 0; k < f.n_keys; k++) {
      const uint32_t code = (uint32_t(s) / f.stride[k]) % f.radix[k];
      reinterpret_cast<uint32_t*>(f.out + 256 + size_t(k) * key_bytes)[o] = code ? code - 1u : 0xffffffffu;
      if (!code) hdr[16 + k] = 1u;
    }
    long long* aggs = reinterpret_cast<long long*>(f.out + 256 + size_t(f.n_keys) * key_bytes);
    long long lo = 0;  // a Unique's UC_LO cell, written with its UC_HI cell (f.out may be page-locked: never read back)
    for (uint32_t a = 0; a < f.n_aggs; a++) {
      long long v;
      if (f.n_src > 0) {
        if (f.agg_pos[a] < 0) {
          v = (long long)rows;
        } else {
          v = agg_identity(f.agg_func[a], f.agg_is_float[a] != 0);
          for (int r = 0; r < f.n_src; r++) {
            if (reinterpret_cast<const unsigned long long*>(f.src[r])[s] == 0) continue;  // an empty group holds the identity, not a value
            v = agg_combine(f.agg_func[a], f.agg_is_float[a] != 0, v, reinterpret_cast<const long long*>(f.src[r] + S * 8 * size_t(1 + f.agg_pos[a]))[s]);
          }
        }
      } else {
        v = f.t_agg[a] ? f.t_agg[a][s] : (long long)rows;
      }
      if (f.agg_unique[a] == UC_LO) {
        lo = v;
      } else if (f.agg_unique[a] == UC_HI) {  // as k_finalize: the value, or NULL (0) with a 0 validity byte in this column
        aggs[size_t(a - 1) * f.max_out + o] = lo == v ? lo : 0;
        reinterpret_cast<uint8_t*>(aggs + size_t(a) * f.max_out)[o] = lo == v;
      } else {
        aggs[size_t(a) * f.max_out + o] = v;
      }
    }
  }
  __shared__ bool last;
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence_system();  // cumulative over the CTA's stores (ordered before it by the barrier): one fence per CTA, not per thread
    last = atomicAdd(hdr + 62, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (last && threadIdx.x < 64) {
    __threadfence();
    uint32_t v = threadIdx.x == 62 ? 0u : atomicAdd(hdr + threadIdx.x, 0u);
    if (threadIdx.x >= 8 && threadIdx.x < 16) v = reinterpret_cast<const uint32_t*>(f.counters)[threadIdx.x - 8];  // counters [0..3] at byte 32
    reinterpret_cast<uint32_t*>(f.out)[threadIdx.x] = v;
    hdr[threadIdx.x] = 0;
  }
}

cudaError_t launch_finalize_dense(const DenseOut& f, cudaStream_t st) {
  k_finalize_dense<<<grid_for(f.table_slots), 256, 0, st>>>(f);
  return cudaGetLastError();
}

cudaError_t launch_merge(const QueryDesc& q, const void* partial, size_t src_slots, cudaStream_t st) {
  k_merge<<<grid_for(src_slots), 256, 0, st>>>(q, static_cast<const uint8_t*>(partial), src_slots);
  return cudaGetLastError();
}

// ---- PLAIN pages: raw chunk bytes -> dense value array (one CTA per page, unaligned source) ----
__global__ void k_gather_pages(const uint8_t* __restrict__ stage, uint8_t* __restrict__ image, const PageCopy* __restrict__ table) {
  const PageCopy c = table[blockIdx.x];
  const uint8_t* src = stage + c.src_off;
  const uint32_t a = uint32_t(reinterpret_cast<uintptr_t>(src) & 7u);
  const unsigned long long* w = reinterpret_cast<const unsigned long long*>(src - a);
  unsigned long long* out = reinterpret_cast<unsigned long long*>(image + c.dst_off);
  const uint64_t n = c.len >> 3;
  if (a == 0) {
    for (uint64_t i = threadIdx.x; i < n; i += blockDim.x) out[i] = w[i];
  } else {
    const uint32_t sh = a * 8u;
    for (uint64_t i = threadIdx.x; i < n; i += blockDim.x) out[i] = (w[i] >> sh) | (w[i + 1] << (64u - sh));  // (the span has 16 bytes of slack)
  }
}

cudaError_t launch_gather_pages(const void* stage, void* image, const PageCopy* table, uint32_t n, cudaStream_t st) {
  if (n == 0) return cudaSuccess;
  k_gather_pages<<<n, 256, 0, st>>>(static_cast<const uint8_t*>(stage), static_cast<uint8_t*>(image), table);
  return cudaGetLastError();
}

// ---- cursor seeds from an uploaded run directory (one thread per 128-row chunk, binary search) ----
// Same result as the host's make_seeds (part_store.cpp): the run that holds the chunk's first value.
__global__ void k_make_seeds(uint8_t* base, const SeedJob* jobs) {
  const SeedJob j = jobs[blockIdx.y];
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= j.n_chunks) return;
  const Run* runs = reinterpret_cast<const Run*>(base + j.runs_off);
  const uint32_t* val0 = j.val0_off == ~0ull ? nullptr : reinterpret_cast<const uint32_t*>(base + j.val0_off);
  const uint32_t v0 = val0 ? val0[t] : t * uint32_t(kIndexRows);
  const uint32_t first = j.is_def ? t * uint32_t(kIndexRows) : v0;
  Seed sd{};
  sd.val0 = v0;
  if (j.n_runs == 0 || first >= j.total) {  // nothing left to decode from this chunk on
    sd.k = j.n_runs;
    sd.start = j.total;
    sd.end = 0xffffffffu;
  } else {
    uint32_t lo = 0, hi = j.n_runs;  // last run with start <= first
    while (hi - lo > 1) {
      const uint32_t mid = (lo + hi) >> 1;
      if (runs[mid].start <= first) lo = mid;
      else hi = mid;
    }
    const Run r = runs[lo];
    sd.k = lo;
    sd.start = r.start;
    sd.end = runs[lo + 1].start;  // the sentinel's start is the total
    sd.off = r.off;
    sd.val = r.val;
    sd.meta = r.meta;
  }
  reinterpret_cast<Seed*>(base + j.seeds_off)[t] = sd;
}

cudaError_t launch_make_seeds(void* image, uint64_t jobs_off, uint32_t n_jobs, uint32_t max_chunks, cudaStream_t st) {
  if (n_jobs == 0 || max_chunks == 0) return cudaSuccess;
  dim3 grid((max_chunks + 255) / 256, n_jobs);
  k_make_seeds<<<grid, 256, 0, st>>>(static_cast<uint8_t*>(image), reinterpret_cast<const SeedJob*>(static_cast<uint8_t*>(image) + jobs_off));
  return cudaGetLastError();
}

// Index of the last job whose first_block <= blk (jobs ascending by first_block).
template <typename Job>
__device__ __forceinline__ uint32_t job_of_block(const Job* jobs, uint32_t n_jobs, uint32_t blk) {
  uint32_t lo = 0, hi = n_jobs;
  while (hi - lo > 1) {
    const uint32_t mid = (lo + hi) >> 1;
    if (__ldg(&jobs[mid].first_block) <= blk) lo = mid; else hi = mid;
  }
  return lo;
}

// ======================================================================================================
// k_flatten: dictionary column chunk -> flat code array (one warp per 128-row block).
//   code = global dictionary id (+ 1 when the chunk has NULLs, 0 = NULL), w = 8, 16 or 32 bits per row.
// Runs once per (part, column) on the device, from the resident hybrid image; the tile-aggregate kernel
// then stages any tile of the column with ONE bulk copy (tile_agg.cu).
// ======================================================================================================
__global__ void __launch_bounds__(NT) k_flatten(const FlatJob* __restrict__ jobs, uint32_t n_jobs, uint32_t total_blocks) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (uint32_t blk = blockIdx.x * NWARP + warp; blk < total_blocks; blk += gridDim.x * NWARP) {
    const FlatJob& J = jobs[job_of_block(jobs, n_jobs, blk)];
    const uint32_t chunk = blk - J.first_block, c0 = chunk * kIndexRows, w = J.w;
    DictReader rd;
    rd.init(J.chunk, chunk, lane);
    uint32_t gid[STEPS];
#pragma unroll
    for (int j = 0; j < STEPS; j++) gid[j] = rd.next(c0 + j * 32 + lane, J.chunk.n_rows);
#pragma unroll
    for (int j = 0; j < STEPS; j++) {
      const uint32_t code = (gid[j] == kNullIdx) ? 0u : gid[j] + 1u - J.bias;  // rows past the end: 0 (padding)
      const uint32_t r = c0 + j * 32 + lane;
      if (w == 8) J.out[r] = uint8_t(code);
      else if (w == 16) reinterpret_cast<uint16_t*>(J.out)[r] = uint16_t(code);
      else reinterpret_cast<uint32_t*>(J.out)[r] = code;
    }
  }
}

cudaError_t launch_flatten(const FlatJob* d_jobs, uint32_t n_jobs, uint32_t total_blocks, int sm_count, cudaStream_t st) {
  if (n_jobs == 0 || total_blocks == 0) return cudaSuccess;
  uint32_t grid = (total_blocks + NWARP - 1) / NWARP;
  if (grid > uint32_t(sm_count) * 8) grid = uint32_t(sm_count) * 8;
  k_flatten<<<grid, NT, 0, st>>>(d_jobs, n_jobs, total_blocks);
  return cudaGetLastError();
}

// ======================================================================================================
// Frame-of-reference and prefix-sum images of PLAIN int64 chunks for the sorted-run kernels (runs_tma.cu,
// runs_prefix.cu).
//   k_chunk_minmax: min / max of every job's chunk into mm[2 j], mm[2 j + 1] (preset to INT64_MAX / INT64_MIN), and
//                   the wrapping sum of every block into bsum[block].
//   k_narrow:       out[r] = uint{8,16,32}(src[r] - base) for the jobs whose range fits 32 bits; pre[r] = the wrapping
//                   sum of src[0 .. r) for the jobs that want a prefix image (the block's offset is the sum of the
//                   block sums before it).
// One CTA per kNarrowRows-row block of one job.
// ======================================================================================================
__global__ void __launch_bounds__(NT) k_chunk_minmax(const NarrowJob* __restrict__ jobs, uint32_t n_jobs, long long* mm,
                                                     unsigned long long* bsum) {
  __shared__ long long s_lo[NWARP], s_hi[NWARP];
  __shared__ unsigned long long s_sum[NWARP];
  const uint32_t j = job_of_block(jobs, n_jobs, blockIdx.x);
  const NarrowJob& J = jobs[j];
  const uint32_t r0 = (blockIdx.x - J.first_block) * kNarrowRows, r1 = min(J.n_rows, r0 + kNarrowRows);
  long long lo = LLONG_MAX, hi = LLONG_MIN;
  unsigned long long sum = 0;
  for (uint32_t r = r0 + threadIdx.x; r < r1; r += NT) {
    const long long v = __ldg(J.src + r);
    lo = min(lo, v);
    hi = max(hi, v);
    sum += (unsigned long long)v;
  }
  for (int o = 16; o; o >>= 1) {
    lo = min(lo, __shfl_xor_sync(0xffffffffu, lo, o));
    hi = max(hi, __shfl_xor_sync(0xffffffffu, hi, o));
    sum += __shfl_xor_sync(0xffffffffu, sum, o);
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) {
    s_lo[warp] = lo;
    s_hi[warp] = hi;
    s_sum[warp] = sum;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < NWARP; w++) {
      lo = min(lo, s_lo[w]);
      hi = max(hi, s_hi[w]);
      sum += s_sum[w];
    }
    atomicMin(mm + 2 * j, lo);
    atomicMax(mm + 2 * j + 1, hi);
    bsum[blockIdx.x] = sum;
  }
}

// exclusive sum over the CTA of one value per thread (wrapping); also returns the CTA total
__device__ __forceinline__ unsigned long long cta_exclusive_sum(unsigned long long v, unsigned long long* s_warp, unsigned long long* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned long long inc = v;
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned long long t = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += t;
  }
  if (lane == 31) s_warp[warp] = inc;
  __syncthreads();
  unsigned long long before = 0, all = 0;
  for (int w = 0; w < NWARP; w++) {
    const unsigned long long t = s_warp[w];
    before += w < warp ? t : 0ull;
    all += t;
  }
  __syncthreads();  // s_warp is reused by the next call
  *total = all;
  return before + inc - v;
}

__global__ void __launch_bounds__(NT) k_narrow(const NarrowJob* __restrict__ jobs, uint32_t n_jobs, const unsigned long long* __restrict__ bsum) {
  __shared__ unsigned long long s_warp[NWARP];
  const NarrowJob& J = jobs[job_of_block(jobs, n_jobs, blockIdx.x)];
  const uint32_t blk = blockIdx.x - J.first_block;
  const uint32_t r0 = blk * kNarrowRows, r1 = min(J.n_rows, r0 + kNarrowRows), w = J.w;
  const unsigned long long base = (unsigned long long)J.base;
  long long* const pre = J.pre;
  unsigned long long carry = 0;  // prefix image: the wrapping sum of the rows before the current step
  if (pre) {
    unsigned long long t = 0;
    for (uint32_t b = threadIdx.x; b < blk; b += NT) t += __ldg(bsum + J.sum_block + b);
    cta_exclusive_sum(t, s_warp, &carry);
  }
  for (uint32_t s = r0; s < r1; s += NT) {  // uniform trip count: the prefix steps synchronise the CTA
    const uint32_t r = s + threadIdx.x;
    const unsigned long long v = r < r1 ? (unsigned long long)__ldg(J.src + r) : 0ull;
    if (w && r < r1) {
      const unsigned long long d = v - base;  // < 2^(8 w): the host chose w from the range
      if (w == 1) J.out[r] = uint8_t(d);
      else if (w == 2) reinterpret_cast<uint16_t*>(J.out)[r] = uint16_t(d);
      else reinterpret_cast<uint32_t*>(J.out)[r] = uint32_t(d);
    }
    if (pre) {
      unsigned long long step = 0;
      const unsigned long long ex = cta_exclusive_sum(v, s_warp, &step);
      if (r < r1) pre[r] = (long long)(carry + ex);
      carry += step;
    }
  }
  if (pre && r1 == J.n_rows && threadIdx.x == 0) pre[r1] = (long long)carry;  // P[n]: the chunk's sum
}

cudaError_t launch_chunk_minmax(const NarrowJob* d_jobs, uint32_t n_jobs, uint32_t total_blocks, long long* d_mm, unsigned long long* d_bsum,
                                cudaStream_t st) {
  if (n_jobs == 0 || total_blocks == 0) return cudaSuccess;
  k_chunk_minmax<<<total_blocks, NT, 0, st>>>(d_jobs, n_jobs, d_mm, d_bsum);
  return cudaGetLastError();
}

cudaError_t launch_narrow(const NarrowJob* d_jobs, uint32_t n_jobs, uint32_t total_blocks, const unsigned long long* d_bsum, cudaStream_t st) {
  if (n_jobs == 0 || total_blocks == 0) return cudaSuccess;
  k_narrow<<<total_blocks, NT, 0, st>>>(d_jobs, n_jobs, d_bsum);
  return cudaGetLastError();
}

cudaError_t launch_decode(const ChunkDesc& c, int32_t* out_i32, long long* out_i64, uint8_t* out_valid, int sm_count,
                          cudaStream_t st) {
  uint32_t n_chunks = (c.n_rows + kIndexRows - 1) / kIndexRows;
  if (n_chunks == 0) return cudaSuccess;
  uint32_t grid = (n_chunks + NWARP - 1) / NWARP;
  if (grid > uint32_t(sm_count) * 8) grid = uint32_t(sm_count) * 8;
  k_decode<<<grid, NT, 0, st>>>(c, n_chunks, out_i32, out_i64, out_valid);
  return cudaGetLastError();
}

}  // namespace fgpu
