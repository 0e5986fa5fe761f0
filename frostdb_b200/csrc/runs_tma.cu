// k_runs_tma: scan + range filter + group-by aggregate for row groups of SORTED parts, CTA-cooperative
// with TMA-staged column tiles (sm_90a).  The plan shape:
//   * the filter is a conjunction of <= 2 int64 range leaves on PLAIN non-null columns and <= 2 dictionary-column
//     leaves on run-length columns (physicalplan/filter.go:276-323, binaryscalarexpr.go:41-311),
//   * every group key is a dictionary-string column that is run-length only in the row group (what compaction
//     leaves behind: rows sorted by the key columns, table.go:1296-1346),
//   * every stored aggregate is Sum / Min / Max over a PLAIN non-null column (aggregate.go:386-560).
//
// Structure: kRtConsumerWarps consumer warps + ONE producer warp per CTA, two CTAs per SM.
//   producer  walks the CTA's tiles (block_rows consecutive rows of one row group).  For every tile it waits until
//             the consumers released the ring stage, issues ONE TMA bulk copy per staged column
//             (cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes, rows x 1, 2, 4 or 8 bytes: the chunk's
//             frame-of-reference image when its range fits 32 bits, see ensure_narrow) and then stages the
//             piece of every key column's run directory that covers the tile: dir_entries entries from the run
//             that holds the tile's first row (found through the 128-row seed), each reduced to
//             {end row of the run, dense-table contribution (id + 1) * stride} — for a dictionary LEAF column
//             {end row, does the leaf pass on this run} (the leaf's result byte per dictionary id is looked up here,
//             once per run and tile, never per row).  One arrive.expect_tx publishes the stage.
//   consumers wait on the stage's `full` mbarrier.  Warp w owns rows [w, w + 1) * block_rows / kRtConsumerWarps
//             of the tile: it finds its first run in the staged directory with one ballot per 32 entries, then walks
//             SEGMENTS — stretches of rows up to the nearest run end of any cursor column, i.e. rows of ONE group.
//             A segment is read with steps aligned to ITS first row (lane i reads row a + 32 s + i: conflict-free
//             1-, 2-, 4- or 8-byte shared loads at any alignment, widened to base + v in 64 bits before the range test
//             and the aggregate), so only its last step is masked, and in row groups whose filter
//             was decided by the chunk statistics the row count of a segment is its length.  Partial sums stay in
//             registers per lane while the group does not change; a change costs three REDUX (22-bit pieces of the
//             64-bit lane sums), and one atomic per aggregate into the dense table in L2.
//             Cursor moves read the staged directory (shared memory), never global memory, except in tiles that
//             hold more runs than dir_entries (global fallback, same result).
//
// Algorithmic bytes per row: the staged width of every distinct staged column (the run directories are O(groups)).
#include <cuda_runtime.h>
#include <cstdio>

#include <algorithm>

#include "agg_ops.cuh"
#include "device_types.h"
#include "kernels.h"
#include "ptx.cuh"

namespace fgpu {
namespace {

constexpr unsigned FULL = 0xffffffffu;
constexpr uint32_t kNoSlot = 0xffffffffu;
constexpr int kNQ = kRunsKeys + kRunsPreds;  // most cursor columns of one launch

__device__ __forceinline__ uint2 lds_v2(uint32_t a) {
  uint2 v;
  asm volatile("ld.shared.v2.b32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(a));
  return v;
}
// one staged value of 1 << LG bytes, zero-extended
template <uint32_t LG>
__device__ __forceinline__ unsigned long long ldsw(uint32_t a) {
  if constexpr (LG == 3) return lds64(a);
  else if constexpr (LG == 2) return lds32(a);
  else if constexpr (LG == 1) return lds16(a);
  else return lds8(a);
}
__device__ __forceinline__ unsigned long long ldsw(uint32_t a, uint32_t lg) {  // lg warp-uniform
  if (lg == 3) return lds64(a);
  if (lg == 2) return lds32(a);
  if (lg == 1) return lds16(a);
  return lds8(a);
}
template <uint32_t V>
struct Lg {
  static constexpr uint32_t value = V;
};
__device__ __forceinline__ void sts_v2(uint32_t a, uint32_t x, uint32_t y) {
  asm volatile("st.shared.v2.b32 [%0], {%1, %2};" ::"r"(a), "r"(x), "r"(y) : "memory");
}
__device__ __forceinline__ void sts32(uint32_t a, uint32_t x) { asm volatile("st.shared.b32 [%0], %1;" ::"r"(a), "r"(x) : "memory"); }

// Cursor column q of a row group: keys first, then the dictionary leaves.
struct CursorCol {
  const Run* runs;  // row-space directory (+ sentinel); null: a leaf decided for this row group (passes everywhere)
  const Seed* seeds;
  const uint8_t* lut;  // leaves: result byte per GLOBAL dictionary id
  uint32_t n_runs;
};
__device__ __forceinline__ CursorCol cursor_col(const RunsRg* R, int q, int nk) {
  CursorCol c;
  if (q < nk) {
    c.runs = ldg_ptr(&R->runs[q]);
    c.seeds = ldg_ptr(&R->seeds[q]);
    c.lut = nullptr;
    c.n_runs = __ldg(&R->n_runs[q]);
  } else {
    c.runs = ldg_ptr(&R->pred_runs[q - nk]);
    c.seeds = ldg_ptr(&R->pred_seeds[q - nk]);
    c.lut = ldg_ptr(&R->pred_lut[q - nk]);
    c.n_runs = __ldg(&R->pred_n_runs[q - nk]);
  }
  return c;
}
// {end row, contribution} of directory entry idx (clamped to the sentinel: never ends)
__device__ __forceinline__ uint2 dir_entry(const CursorCol& c, uint32_t idx, bool is_key, uint32_t stride, uint32_t pred_null) {
  if (c.runs == nullptr) return make_uint2(0xffffffffu, 1u);
  if (idx >= c.n_runs) return make_uint2(0xffffffffu, 0u);
  const uint32_t val = __ldg(&c.runs[idx].val);
  const uint32_t end = __ldg(&c.runs[idx + 1].start);
  uint32_t con;
  if (is_key) con = (val + 1u) * stride;  // NULL (0xffffffff) contributes 0
  else con = (val == 0xffffffffu) ? pred_null : uint32_t(__ldg(c.lut + val));
  return make_uint2(end, con);
}
// Slow path of a consumer cursor (the tile holds more runs than the staged window): entry k0 + rel from global memory;
// rel == 0xffffffff: the entry that holds `row`, found through the seed.  Returns {end, contribution, rel}.
__device__ __noinline__ uint3 cursor_global(const RunsRg* R, int q, int nk, uint32_t stride, uint32_t pred_null, uint32_t k0, uint32_t rel,
                                            uint32_t row) {
  const CursorCol c = cursor_col(R, q, nk);
  uint32_t idx = k0 + rel;
  if (rel == 0xffffffffu) {
    idx = c.runs ? __ldg(&c.seeds[row / uint32_t(kIndexRows)].k) : 0u;
    while (c.runs && idx < c.n_runs && __ldg(&c.runs[idx + 1].start) <= row) idx++;  // (the seed names the run of the chunk's first row)
  }
  const uint2 e = dir_entry(c, idx, q < nk, stride, pred_null);
  return make_uint3(e.x, e.y, idx - k0);
}

// stage header (144 bytes): k0 of every cursor column, then the tile itself, then the staged columns' layout
constexpr uint32_t kHdrCnt = 20;                           // directory entries staged for every cursor column (0: a decided leaf)
constexpr uint32_t kHdrR0 = 40, kHdrN = 44, kHdrRg = 48, kHdrT = 52;  // first row inside the row group; rows (0: no more tiles); row group; its tile rows
constexpr uint32_t kHdrCol = 64;  // staged column c: {byte offset in the column region, log2 bytes per row, base (8 bytes)} at kHdrCol + 16 c
constexpr uint32_t kHdrBytes = kHdrCol + 16u * kRunsCols;
__device__ __forceinline__ uint4 lds_v4(uint32_t a) {
  uint4 v;
  asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(a));
  return v;
}
// base + the staged value of column c in row r (col: the lane's address of row 0); the layout is read from the stage
// header per use, so that neither the width nor the base of any column occupies registers across the loops
__device__ __forceinline__ unsigned long long col_value(uint32_t stage_s, uint32_t c, uint32_t col, uint32_t r) {
  const uint4 m = lds_v4(stage_s + kHdrCol + 16u * c);
  return ((unsigned long long)m.z | ((unsigned long long)m.w << 32)) + ldsw(col + (r << m.y), m.y);
}

// GEN = false: every stored aggregate is Sum(int64).  GEN = true: Sum / Min / Max over int64 or float64 (agg_ops.cuh).
// HP: the launch has dictionary leaves (cursor columns behind the keys).
template <int NL, int NK, int NA, bool GEN, bool HP>
__global__ void __launch_bounds__(kRtMaxThreads, 3) k_runs_tma(const __grid_constant__ RunsDesc d) {
  extern __shared__ __align__(128) uint8_t dyn[];
  constexpr int NQ = HP ? kNQ : NK;  // cursor columns the code is unrolled for
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t S = d.n_ring, E = d.dir_entries, n_cols = d.n_cols;
  const uint32_t n_pred = HP ? d.n_pred : 0u;
  const uint32_t kW = d.n_consumers;
  const uint32_t dir_bytes = E * 16u;
  const uint32_t bars = smem_u32(dyn);
  const uint32_t stage0 = bars + 128u;  // stage: [header 64][directories kNQ x E x 16][columns at RunsRg::col_soff]

  if (tid == 0) {
    for (uint32_t s = 0; s < S; s++) {
      mbar_init(bars + s * 8, 1);         // full: the producer's expect_tx arrive
      mbar_init(bars + (S + s) * 8, kW);  // empty: one arrive per consumer warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (uint32_t(warp) == kW) {
    // ================================ producer warp ================================
    // The CTA takes tiles b, b + G, ... of the launch's tile table {row group, first row}.  Everything a tile needs
    // hangs on a chain of dependent global loads: table entry -> the row group's pointers -> the 128-row seeds that
    // name the first / last run of the tile -> (TMA) the directory slices and the column data.  The chain is software
    // pipelined over four tiles: every iteration issues the loads of one link for one tile and consumes what the
    // previous iteration issued, so no link's latency is ever waited for.  Lane q owns cursor column q (its pointers
    // and seeds), lane c the pointer of staged column c; lane 0 issues the copies.
    const uint2* const tiles = reinterpret_cast<const uint2*>(d.rg_first_span);
    const uint32_t G = gridDim.x, n_tiles = d.n_spans, CH = d.span_blocks;
    const uint32_t nq = uint32_t(NK) + n_pred;
    // tile sequence: chunks of CH consecutive table entries (consecutive rows: a warp's running group survives from
    // one tile to the next when runs are long); chunk b first, further chunks by ticket (counters[2], zeroed with the
    // table) — requested when a chunk starts, consumed when it ends
    unsigned int* const ticket = reinterpret_cast<unsigned int*>(d.counters + 2);
    uint32_t ch_base = blockIdx.x * CH, ch_pos = 0, next_raw = 0;
    if (lane == 0) next_raw = atomicAdd(ticket, 1u);
    auto next_tile = [&]() -> uint32_t {
      const uint32_t t = ch_base + ch_pos;
      if (++ch_pos == CH) {
        ch_pos = 0;
        ch_base = (G + __shfl_sync(FULL, next_raw, 0)) * CH;
        if (lane == 0) next_raw = atomicAdd(ticket, 1u);
      }
      return t;
    };
    struct Ctx {
      uint32_t tile;      // index into the tile table (>= n_tiles: none)
      uint32_t rg, r0;    // link 1
      const Run* runs;    // link 2: this lane's cursor column (lane < nq), null: decided leaf
      const Seed* seeds;
      const uint8_t* col;  // this lane's staged column (lane < n_cols), null: not staged in this row group
      uint32_t col_sl;     // its RunsCol: soff | lg << 24
      uint32_t n_runs, n_rows, T;
      uint32_t k0, k1;    // link 3: runs that hold the tile's first row and the first row behind the tile
    };
    auto link1 = [&](Ctx& c) {
      c.tile = next_tile();
      if (c.tile < n_tiles) {
        const uint2 t = __ldg(tiles + c.tile);
        c.rg = t.x;
        c.r0 = t.y;
      }
    };
    auto link2 = [&](Ctx& c) {
      c.runs = nullptr;
      c.seeds = nullptr;
      c.col = nullptr;
      c.col_sl = 0;
      c.n_runs = 0;
      c.n_rows = 0;
      c.T = 0;
      if (c.tile < n_tiles) {
        const RunsRg* R = d.rgs + c.rg;
        c.n_rows = __ldg(&R->n_rows);
        c.T = __ldg(&R->tile_rows);
        if (uint32_t(lane) < nq) {
          const int qk = lane < NK ? lane : 0, qp = lane >= NK ? lane - NK : 0;
          c.runs = lane < NK ? ldg_ptr(&R->runs[qk]) : ldg_ptr(&R->pred_runs[qp]);
          c.seeds = lane < NK ? ldg_ptr(&R->seeds[qk]) : ldg_ptr(&R->pred_seeds[qp]);
          c.n_runs = lane < NK ? __ldg(&R->n_runs[qk]) : __ldg(&R->pred_n_runs[qp]);
        }
        if (uint32_t(lane) < n_cols) {
          c.col = ldg_ptr(&R->col[lane]);
          const uint2 sl = __ldg(reinterpret_cast<const uint2*>(&R->cl[lane]));
          c.col_sl = sl.x | (sl.y << 24);
        }
      }
    };
    auto link3 = [&](Ctx& c) {
      c.k0 = 0;
      c.k1 = 0;
      if (c.tile < n_tiles && c.runs != nullptr) {
        const uint32_t behind = c.r0 + c.T;
        c.k0 = __ldg(&c.seeds[c.r0 / uint32_t(kIndexRows)].k);
        c.k1 = behind < c.n_rows ? __ldg(&c.seeds[behind / uint32_t(kIndexRows)].k) : c.n_runs - 1u;
      }
    };
    Ctx c0, c1, c2, c3;
    link1(c0); link1(c1); link1(c2); link1(c3);
    link2(c0); link2(c1); link2(c2);
    link3(c0); link3(c1);
    uint32_t st = 0, ph = 0, n_it = 0;
    for (;;) {
      if (n_it >= S) mbar_wait(bars + (S + st) * 8, ph ^ 1u);  // the consumers are done with the tile that lived here
      const uint32_t stage_s = stage0 + st * d.stage_bytes;
      const uint32_t full = bars + st * 8;
      if (c0.tile >= n_tiles) {  // end marker: a tile without rows
        if (lane == 0) {
          sts32(stage_s + kHdrN, 0u);
          mbar_arrive(full);
        }
        break;
      }
      const uint32_t n = min(c0.T, c0.n_rows - c0.r0);
      uint32_t bytes = 0;
#pragma unroll
      for (int c = 0; c < kRunsCols; c++) {
        if (uint32_t(c) < n_cols) {
          const unsigned long long colc = __shfl_sync(FULL, reinterpret_cast<unsigned long long>(c0.col), c);
          const uint32_t sl = __shfl_sync(FULL, c0.col_sl, c), lg = sl >> 24;
          if (lane == 0 && colc != 0ull) {
            const uint32_t cb = ((n << lg) + 15u) & ~15u;  // (images and extents keep >= 16 readable bytes behind the last row)
            bulk_g2s(stage_s + d.col_off + (sl & 0xffffffu), reinterpret_cast<const uint8_t*>(colc) + (size_t(c0.r0) << lg), cb, full);
            bytes += cb;
          }
        }
      }
      if (lane == 0 && n_cols) {  // the columns' layout {soff, lg, base} for the consumers: RunsRg::cl
        bulk_g2s(stage_s + kHdrCol, d.rgs[c0.rg].cl, n_cols * 16u, full);
        bytes += n_cols * 16u;
      }
      // directory slices: entries k0 .. k1 + 1 of every cursor column (the entry behind the last run carries its end)
#pragma unroll
      for (int q = 0; q < NQ; q++) {
        if (q < NK || uint32_t(q - NK) < n_pred) {
          const unsigned long long rq = __shfl_sync(FULL, reinterpret_cast<unsigned long long>(c0.runs), q);
          const uint32_t k0 = __shfl_sync(FULL, c0.k0, q), k1 = __shfl_sync(FULL, c0.k1, q);
          if (lane == 0) {
            const uint32_t cnt = rq ? min(E, k1 - k0 + 2u) : 0u;
            if (cnt) {
              bulk_g2s(stage_s + kHdrBytes + uint32_t(q) * dir_bytes, reinterpret_cast<const Run*>(rq) + k0, cnt * 16u, full);
              bytes += cnt * 16u;
            }
            sts32(stage_s + uint32_t(q) * 4u, k0);
            sts32(stage_s + kHdrCnt + uint32_t(q) * 4u, cnt);
          }
        }
      }
      if (lane == 0) {
        sts32(stage_s + kHdrR0, c0.r0);
        sts32(stage_s + kHdrN, n);
        sts32(stage_s + kHdrRg, c0.rg);
        sts32(stage_s + kHdrT, c0.T);
        mbar_expect_tx(full, bytes);  // release: the header stores above are visible to the waiters
      }
      __syncwarp();
      // rotate the pipeline: every context moves one link further
      c0 = c1;
      c1 = c2;
      link3(c1);
      c2 = c3;
      link2(c2);
      link1(c3);
      n_it++;
      if (++st == S) {
        st = 0;
        ph ^= 1u;
      }
    }
  } else {
    // ================================ consumer warps ================================
    uint32_t cs = kNoSlot, cnt = 0, ucnt = 0;
    bool counted = false;  // per-lane counts pending (rows of a filtered segment since the last flush)
    unsigned long long sel = 0;
    unsigned long long part[NA > 0 ? NA : 1];
    uint32_t afunc[NA > 0 ? NA : 1];
    bool aflt[NA > 0 ? NA : 1];
#pragma unroll
    for (int a = 0; a < NA; a++) {
      afunc[a] = GEN ? (d.agg_func[a] & 0xffu) : 1u;
      aflt[a] = GEN && (d.agg_func[a] >> 8) != 0;
      part[a] = GEN ? (unsigned long long)agg_identity(uint8_t(afunc[a]), aflt[a]) : 0ull;
    }
    // lane 0 adds the row count, lane 1 + a the sum of aggregate a: ONE atomic instruction per group change
    unsigned long long* const my_cell = lane == 0 ? d.t_rows : reinterpret_cast<unsigned long long*>(d.t_agg[(lane >= 1 && lane <= NA) ? lane - 1 : 0]);
    auto fold = [&](int q, bool act, unsigned long long v) {
      if constexpr (GEN) {
        if (act) part[q] = (unsigned long long)agg_combine(uint8_t(afunc[q]), aflt[q], (long long)part[q], (long long)v);
      } else {
        part[q] += act ? v : 0ull;
      }
    };
    auto flush = [&]() {
      uint32_t tt = ucnt;
      if (NL > 0 && counted) tt += __reduce_add_sync(FULL, cnt);
      ucnt = 0;
      cnt = 0;
      counted = false;
      if (tt == 0) return;  // a group that received no row leaves the table untouched
      sel += tt;
      if constexpr (GEN) {
        if (lane == 0) atomicAdd(d.t_rows + cs, (unsigned long long)tt);
#pragma unroll
        for (int a = 0; a < NA; a++) {
          unsigned long long v = part[a];
#pragma unroll
          for (int o = 16; o; o >>= 1)
            v = (unsigned long long)agg_combine(uint8_t(afunc[a]), aflt[a], (long long)v, (long long)__shfl_xor_sync(FULL, v, o));
          if (lane == 0) apply_agg(uint8_t(afunc[a]), aflt[a], d.t_agg[a] + cs, (long long)v);
          part[a] = (unsigned long long)agg_identity(uint8_t(afunc[a]), aflt[a]);
        }
      } else {
        unsigned long long mine = tt;
#pragma unroll
        for (int a = 0; a < NA; a++) {
          unsigned long long v = part[a];
          part[a] = 0;
          if (!__any_sync(FULL, (v >> 27) != 0ull)) {  // every lane sum below 2^27: one 32-bit REDUX is exact
            v = __reduce_add_sync(FULL, uint32_t(v));
          } else {  // three 32-bit REDUX sums over 22-bit pieces (32 x 2^22 fits): no shuffle chain
            const uint32_t s0 = __reduce_add_sync(FULL, uint32_t(v) & 0x3fffffu);
            const uint32_t s1 = __reduce_add_sync(FULL, uint32_t(v >> 22) & 0x3fffffu);
            const uint32_t s2 = __reduce_add_sync(FULL, uint32_t(v >> 44));
            v = (unsigned long long)s0 + ((unsigned long long)s1 << 22) + ((unsigned long long)s2 << 44);
          }
          if (lane == a + 1) mine = v;
        }
        if (lane <= NA) atomicAdd(my_cell + cs, mine);
      }
    };

    uint32_t rg_cached = 0xffffffffu;
    long long lo[NL > 0 ? NL : 1], hi[NL > 0 ? NL : 1];
    bool all_pass = NL == 0;
    uint32_t stride[NK > 0 ? NK : 1];
#pragma unroll
    for (int k = 0; k < NK; k++) stride[k] = d.stride[k];
    const uint8_t* plut[kRunsPreds] = {nullptr, nullptr};  // result byte per GLOBAL dictionary id of every dictionary leaf

    uint32_t st = 0, ph = 0;
    for (;;) {
      mbar_wait(bars + st * 8, ph);
      const uint32_t stage_s = stage0 + st * d.stage_bytes;
      const uint32_t n = lds32(stage_s + kHdrN);
      if (n == 0) break;  // the producer's end marker
      const uint32_t r0 = lds32(stage_s + kHdrR0), rg = lds32(stage_s + kHdrRg);
      const RunsRg* const R = d.rgs + rg;
      if (NL > 0 || HP) {
        if (rg != rg_cached) {
          rg_cached = rg;
#pragma unroll
          for (int l = 0; l < NL; l++) {
            lo[l] = __ldg(&R->lo[l]);
            hi[l] = __ldg(&R->hi[l]);
          }
          if (NL > 0) all_pass = __ldg(&R->all_pass) != 0;  // warp-uniform: statistics decided the filter
          if constexpr (HP) {
#pragma unroll
            for (int p = 0; p < kRunsPreds; p++) plut[p] = uint32_t(p) < n_pred ? ldg_ptr(&R->pred_lut[p]) : nullptr;
          }
        }
      }
      const uint32_t T = lds32(stage_s + kHdrT), SUB = T >> d.consumers_log2;
      const uint32_t s0 = r0 + uint32_t(warp) * SUB, s1 = min(r0 + n, s0 + SUB);
      if (s0 < s1) {
        const uint32_t cols_s = stage_s + d.col_off;
        // cursors: the run of every cursor column that holds row s0 (staged entry j = directory entry k0 + j, raw:
        // {first row, -, dictionary id or NULL, -}; the end of a run is the first row of the next entry)
        uint32_t ci[NQ > 0 ? NQ : 1], cend[NQ > 0 ? NQ : 1], ccon[NQ > 0 ? NQ : 1], ccnt[NQ > 0 ? NQ : 1];
        auto entry = [&](int q) {  // loads cend / ccon of cursor q at ci[q]
          const uint32_t dq = stage_s + kHdrBytes + uint32_t(q) * dir_bytes + ci[q] * 16u;
          if (ci[q] + 1u < ccnt[q]) {
            const uint32_t val = lds32(dq + 8u);
            cend[q] = lds32(dq + 16u);
            if (q < NK) ccon[q] = (val + 1u) * stride[q < NK ? q : 0];  // NULL (0xffffffff) contributes 0
            else ccon[q] = val == 0xffffffffu ? d.pred_null[q >= NK ? q - NK : 0] : uint32_t(__ldg(plut[q >= NK ? q - NK : 0] + val));
          } else {  // the tile holds more runs than the staged window
            const uint3 g = cursor_global(R, q, NK, q < NK ? stride[q < NK ? q : 0] : 0u, q < NK ? 0u : d.pred_null[q >= NK ? q - NK : 0],
                                          lds32(stage_s + uint32_t(q) * 4u), ci[q], 0u);
            cend[q] = g.x;
            ccon[q] = g.y;
          }
        };
#pragma unroll
        for (int q = 0; q < NQ; q++) {
          ci[q] = 0;
          cend[q] = 0xffffffffu;
          ccon[q] = q < NK ? 0u : 1u;
          ccnt[q] = 0;
          if (q < NK || uint32_t(q - NK) < n_pred) {
            ccnt[q] = lds32(stage_s + kHdrCnt + uint32_t(q) * 4u);
            if (ccnt[q]) {
              const uint32_t dq = stage_s + kHdrBytes + uint32_t(q) * dir_bytes;
              uint32_t idx = 0;
              for (uint32_t b = 0; b < ccnt[q]; b += 32u) {
                const uint32_t j = b + uint32_t(lane);
                const uint32_t c = __popc(__ballot_sync(FULL, j < ccnt[q] && lds32(dq + j * 16u) <= s0));
                idx += c;
                if (c < 32u) break;
              }
              if (idx < ccnt[q]) {
                ci[q] = idx - 1u;  // entry 0 starts at or before the tile's first row
                entry(q);
              } else {  // the run of s0 lies behind the staged window: found through the seed
                const uint3 g = cursor_global(R, q, NK, q < NK ? stride[q < NK ? q : 0] : 0u, q < NK ? 0u : d.pred_null[q >= NK ? q - NK : 0],
                                              lds32(stage_s + uint32_t(q) * 4u), 0xffffffffu, s0);
                cend[q] = g.x;
                ccon[q] = g.y;
                ci[q] = g.z;
              }
            }
          }
        }
        auto advance = [&](int q) {
          ci[q]++;
          entry(q);
        };
        // staged leaf / aggregate columns: address of row r in lane i = col + (r + i) << lg; value = base + staged
        uint32_t lcol[NL > 0 ? NL : 1], acol[NA > 0 ? NA : 1];
        auto col_addr = [&](uint32_t c) {
          const uint2 m = lds_v2(stage_s + kHdrCol + 16u * c);
          return cols_s + m.x + ((uint32_t(lane) - r0) << m.y);
        };
#pragma unroll
        for (int l = 0; l < NL; l++) lcol[l] = col_addr(d.leaf_col[l]);
#pragma unroll
        for (int a = 0; a < NA; a++) acol[a] = col_addr(d.agg_col[a]);
        // all_pass segment of aggregate q at row `row`: every step unmasked but the last, LG bytes per staged value
        auto fold_seg = [&](int q, uint32_t row, uint32_t whole, uint32_t rem, auto L) {
          constexpr uint32_t LG = decltype(L)::value, stp = 32u << LG;
          const uint2 bw = lds_v2(stage_s + kHdrCol + 16u * d.agg_col[q] + 8u);
          const unsigned long long b = (unsigned long long)bw.x | ((unsigned long long)bw.y << 32);
          uint32_t a0 = acol[q] + (row << LG);
#pragma unroll 1
          for (uint32_t s = whole >> 2; s; s--, a0 += 4u * stp) {
            const unsigned long long v0 = ldsw<LG>(a0), v1 = ldsw<LG>(a0 + stp), v2 = ldsw<LG>(a0 + 2u * stp), v3 = ldsw<LG>(a0 + 3u * stp);
            fold(q, true, b + v0);
            fold(q, true, b + v1);
            fold(q, true, b + v2);
            fold(q, true, b + v3);
          }
          if (whole & 2u) {
            const unsigned long long v0 = ldsw<LG>(a0), v1 = ldsw<LG>(a0 + stp);
            fold(q, true, b + v0);
            fold(q, true, b + v1);
            a0 += 2u * stp;
          }
          if (whole & 1u) {
            fold(q, true, b + ldsw<LG>(a0));
            a0 += stp;
          }
          if (uint32_t(lane) < rem) fold(q, true, b + ldsw<LG>(a0));
        };

        uint32_t row = s0;
        while (row < s1) {
          uint32_t seg_end = s1, us = 0, skip_to = 0;
#pragma unroll
          for (int k = 0; k < NK; k++) {
            seg_end = min(seg_end, cend[k]);
            us += ccon[k];
          }
          if constexpr (HP) {
#pragma unroll
            for (int p = 0; p < kRunsPreds; p++) {
              seg_end = min(seg_end, cend[NK + p]);
              if (ccon[NK + p] == 0u) skip_to = max(skip_to, cend[NK + p]);  // rows of a run that fails a leaf are skipped as a whole
            }
          }
          if (HP && skip_to) {
            seg_end = min(s1, skip_to);
          } else {
            if (us != cs) {
              if (cs != kNoSlot) flush();
              cs = us;
            }
            const uint32_t len = seg_end - row, whole = len >> 5, rem = len & 31u;
            if (all_pass) {
              ucnt += len;
#pragma unroll
              for (int q = 0; q < NA; q++) {
                switch (lds32(stage_s + kHdrCol + 16u * d.agg_col[q] + 4u)) {  // log2 bytes per row (warp-uniform)
                  case 0: fold_seg(q, row, whole, rem, Lg<0>{}); break;
                  case 1: fold_seg(q, row, whole, rem, Lg<1>{}); break;
                  case 2: fold_seg(q, row, whole, rem, Lg<2>{}); break;
                  default: fold_seg(q, row, whole, rem, Lg<3>{}); break;
                }
              }
            } else if (NL > 0) {
              counted = true;
              // whole steps: no row mask; the tail step re-reads the segment's first row in the lanes behind its end
              uint32_t r = row;
#pragma unroll 2
              for (uint32_t s = 0; s < whole; s++, r += 32u) {
                bool in = true;
#pragma unroll
                for (int l = 0; l < NL; l++) {
                  const long long x = (long long)col_value(stage_s, d.leaf_col[l], lcol[l], r);
                  in = in && x >= lo[l] && x <= hi[l];
                }
                if (in) cnt++;
#pragma unroll
                for (int q = 0; q < NA; q++) {
                  const unsigned long long v = col_value(stage_s, d.agg_col[q], acol[q], r);
                  if constexpr (GEN) fold(q, in, v);
                  else if (in) part[q] += v;
                }
              }
              if (rem) {
                bool in = uint32_t(lane) < rem;
                if (!in) r = row - uint32_t(lane);
#pragma unroll
                for (int l = 0; l < NL; l++) {
                  const long long x = (long long)col_value(stage_s, d.leaf_col[l], lcol[l], r);
                  in = in && x >= lo[l] && x <= hi[l];
                }
                if (in) cnt++;
#pragma unroll
                for (int q = 0; q < NA; q++) fold(q, in, col_value(stage_s, d.agg_col[q], acol[q], r));
              }
            }
          }
          row = seg_end;
#pragma unroll
          for (int q = 0; q < NQ; q++)
            if (q < NK || uint32_t(q - NK) < n_pred)
              while (cend[q] <= row) advance(q);
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(bars + (S + st) * 8);
      if (++st == S) {
        st = 0;
        ph ^= 1u;
      }
    }
    if (cs != kNoSlot) flush();
    if (lane == 0 && sel) atomicAdd(d.counters, sel);  // rows that passed the filter
  }
}

using RtKern = void (*)(const RunsDesc);
template <int NL, int NK, bool HP>
RtKern pick_na(int na, bool gen) {
  if (gen && na > 0) return na == 1 ? k_runs_tma<NL, NK, 1, true, HP> : (na == 2 ? k_runs_tma<NL, NK, 2, true, HP> : k_runs_tma<NL, NK, 3, true, HP>);
  switch (na) {
    case 0: return k_runs_tma<NL, NK, 0, false, HP>;
    case 1: return k_runs_tma<NL, NK, 1, false, HP>;
    case 2: return k_runs_tma<NL, NK, 2, false, HP>;
    default: return k_runs_tma<NL, NK, 3, false, HP>;
  }
}
template <int NL, bool HP>
RtKern pick_nk(int nk, int na, bool gen) {
  switch (nk) {
    case 0: return pick_na<NL, 0, HP>(na, gen);
    case 1: return pick_na<NL, 1, HP>(na, gen);
    case 2: return pick_na<NL, 2, HP>(na, gen);
    default: return pick_na<NL, 3, HP>(na, gen);
  }
}
template <bool HP>
RtKern pick_nl(int nl, int nk, int na, bool gen) {
  switch (nl) {
    case 0: return pick_nk<0, HP>(nk, na, gen);
    case 1: return pick_nk<1, HP>(nk, na, gen);
    default: return pick_nk<2, HP>(nk, na, gen);
  }
}
RtKern pick(const RunsDesc& d, int nl, int nk, int na) {
  bool gen = false;  // any reducer other than Sum(int64)
  for (int a = 0; a < na; a++) gen = gen || d.agg_func[a] != 1u;
  return d.n_pred ? pick_nl<true>(nl, nk, na, gen) : pick_nl<false>(nl, nk, na, gen);
}

}  // namespace

// Rows per tile of a row group whose staged columns take row_bytes per row: tile_bytes of column data, a multiple of
// 1024 rows, but not much more than the row group (the stage is sized for the largest tile of the launch) and, where
// runs are short, few enough rows that the tile rarely holds more runs of a cursor column (max_runs in the row group)
// than the staged directory window.
uint32_t runs_tma_tile_rows(uint32_t tile_bytes, uint32_t row_bytes, uint32_t n_rows, uint32_t max_runs) {
  uint64_t t = tile_bytes / std::max<uint32_t>(row_bytes, 1u);
  t = std::min<uint64_t>(t, (uint64_t(n_rows) + 1023u) & ~uint64_t(1023));
  if (max_runs) t = std::min<uint64_t>(t, uint64_t(kRtDirMax) * n_rows / max_runs);
  return uint32_t(std::max<uint64_t>(t & ~uint64_t(1023), 1024u));
}

// Ring depth, consumer warps and stage layout for a launch with nq cursor columns whose largest tile has max_tile rows
// and holds col_region bytes of column data (fills the descriptor).
void runs_tma_plan(RunsDesc& d, int nq, uint32_t max_tile, uint32_t col_region, int force_stages, int force_warps, int force_chunk) {
  uint32_t S = 2;  // two stages of 32 KB leave room for three CTAs per SM: measured faster than deeper rings under two
  if (force_stages >= 2 && force_stages <= 8) S = uint32_t(force_stages);
  uint32_t W = uint32_t(kRtConsumerWarps);
  if (force_warps == 4 || force_warps == 8) W = uint32_t(force_warps);
  d.block_rows = max_tile;
  // one tile per ticket: with 1-2 bytes per staged row a launch has only a few tiles per CTA, and single tiles balance
  // the tail best (DESIGN §7)
  d.span_blocks = force_chunk >= 1 && force_chunk <= 64 ? uint32_t(force_chunk) : 1u;
  d.n_ring = S;
  d.n_consumers = W;
  d.consumers_log2 = W == 4 ? 2u : (W == 8 ? 3u : 4u);
  // staged directory window: max_tile / 32 entries cover a tile whose runs average 32 rows; halved while two CTAs do not fit an SM
  d.dir_entries = std::min<uint32_t>(max_tile / 32u, uint32_t(kRtDirMax));
  for (;;) {
    d.col_off = (kHdrBytes + uint32_t(nq) * d.dir_entries * 16u + 127u) & ~127u;
    d.stage_bytes = d.col_off + ((col_region + 127u) & ~127u);
    if (d.dir_entries <= 32u || 2 * (runs_tma_smem_bytes(d) + 1024) <= 228u * 1024u) break;
    d.dir_entries >>= 1;
  }
  while (d.n_ring > 2 && runs_tma_smem_bytes(d) > 227u * 1024u) d.n_ring--;
}

size_t runs_tma_smem_bytes(const RunsDesc& d) { return 128 + size_t(d.n_ring) * d.stage_bytes; }

int runs_tma_ctas_per_sm(const RunsDesc& d) {
  const size_t per_cta = runs_tma_smem_bytes(d) + 1024;
  int n = int((228u * 1024u) / per_cta);
  const int by_threads = 2048 / int((d.n_consumers + 1) * 32), by_regs = 65536 / int((d.n_consumers + 1) * 32 * 72);
  n = std::min(n, std::min(by_threads, by_regs));
  return std::max(1, std::min(n, 4));
}

cudaError_t launch_runs_tma(const RunsDesc& d, int nl, int nk, int na, int sm_count, cudaStream_t st) {
  if (d.n_spans == 0) return cudaSuccess;
  const size_t smem = runs_tma_smem_bytes(d);
  RtKern kern = pick(d, nl, nk, na);
  const cudaError_t e = kernel_smem_at_least(reinterpret_cast<const void*>(kern), smem);
  if (e != cudaSuccess) return e;
  uint32_t grid = uint32_t(sm_count) * uint32_t(runs_tma_ctas_per_sm(d));
  const uint32_t chunks = (d.n_spans + d.span_blocks - 1) / d.span_blocks;
  if (grid > chunks) grid = chunks;
  kern<<<grid, (d.n_consumers + 1) * 32, smem, st>>>(d);
  return cudaGetLastError();
}

}  // namespace fgpu
