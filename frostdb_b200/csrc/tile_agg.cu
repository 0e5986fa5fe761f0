// k_tile_agg: scan + filter + group-by aggregate for row groups whose key columns are NOT long sorted runs
// (bit-packed dictionary indices of unsorted parts and fresh L0 records, short runs, NULLs) — sm_90a.
//
// Takes over, for those row groups, what TableScan -> PredicateFilter -> HashAggregate do per record in the
// reference (physicalplan/filter.go:276-323, physicalplan/aggregate.go:263-490: per row a hash of the key
// values, a map lookup and an append to the group's buffer), when
//   * the filter is a conjunction of <= kTaLeaves numeric range leaves on PLAIN non-null columns and
//     <= kTaPreds dictionary-column leaves (==, !=, contains, regex, == NULL: one result byte per dictionary id),
//   * every group key is a dictionary-string column (dense mixed-radix table),
//   * every stored aggregate is Sum / Min / Max of a PLAIN non-null int64 or float64 column (Count needs no input).
//
// Structure: one CTA per SM, kTaConsumerWarps consumer warps + ONE producer warp.
//   producer  walks the CTA's tiles (tile_rows consecutive rows of one row group).  For every tile it waits until
//             the consumers released the ring stage, writes the tile header (row group descriptor + row range)
//             into the stage, arms the stage's `full` mbarrier with the byte count and issues ONE TMA bulk copy
//             (cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes) per projected column: 8 KB -
//             32 KB each.  PLAIN columns are 8 bytes per row; dictionary columns are flat code arrays of w bits
//             per row (k_flatten), so a tile of any column is one contiguous 128-byte aligned range.
//   consumers wait on `full`, walk the tile with one row per lane and step (consecutive lanes = consecutive rows:
//             conflict-free 8-byte shared loads, code extraction from at most two 32-bit shared words), evaluate
//             the leaves, compute the dense slot and fold the row into the CTA-private table in shared memory:
//             ATOMS.POPC.INC for the row count, ATOMS.ADD on the low word of an int64 Sum (a carry out of the low
//             word — detected from the returned old value — and the high word go to the global table directly; for
//             values that fit 32 bits that never happens), 64-bit CAS cells for Min / Max / float64.
//             A stage is handed back through the `empty` mbarrier (one arrive per warp).
//   epilogue  every CTA folds its table into the global one (one atomic per occupied slot and aggregate).
// Tables that do not fit shared memory (> ~160 KB) are updated in global memory directly.
//
// Algorithmic bytes per row: 8 per staged PLAIN column + w / 8 per staged code column.
#include <cuda_runtime.h>

#include "agg_ops.cuh"
#include "device_types.h"
#include "kernels.h"
#include "ptx.cuh"

namespace fgpu {
namespace {

constexpr unsigned FULL = 0xffffffffu;
constexpr int NC = kTaConsumerWarps * 32;  // consumer threads
constexpr uint32_t kHdrBytes = 256;        // per-stage tile header: TileAggRg + row range
static_assert(sizeof(TileAggRg) + 16 <= kHdrBytes, "tile header fits its slot");

// Predicated shared-memory atomics (PTX-level predicates keep the row loop free of divergence regions).
__device__ __forceinline__ void red_add_shared_if(uint32_t addr, uint32_t v, bool p) {
  asm volatile(
      "{\n"
      ".reg .pred q;\n"
      "setp.ne.u32 q, %2, 0;\n"
      "@q red.shared.add.u32 [%0], %1;\n"
      "}\n" ::"r"(addr),
      "r"(v), "r"(uint32_t(p))
      : "memory");
}
__device__ __forceinline__ uint32_t atom_add_shared_if(uint32_t addr, uint32_t v, bool p) {
  uint32_t old = 0;
  asm volatile(
      "{\n"
      ".reg .pred q;\n"
      "setp.ne.u32 q, %3, 0;\n"
      "@q atom.shared.add.u32 %0, [%1], %2;\n"
      "}\n"
      : "+r"(old)
      : "r"(addr), "r"(v), "r"(uint32_t(p))
      : "memory");
  return old;
}

// 64-bit cell in shared memory (Min / Max / float64 Sum): compare-and-swap loop, Go's `<` / `>` NaN behaviour
__device__ __forceinline__ void smem_apply64(uint32_t func, bool is_float, unsigned long long* cell, long long v) {
  unsigned long long old = *cell;
  for (;;) {
    const long long nv = agg_combine(uint8_t(func), is_float, (long long)old, v);
    if (nv == (long long)old) return;
    const unsigned long long prev = atomicCAS(cell, old, (unsigned long long)nv);
    if (prev == old) return;
    old = prev;
  }
}

struct TileHdr {  // what the producer leaves in front of every staged tile
  TileAggRg rg;
  uint32_t r0, n;   // first row of the tile inside the row group, rows in the tile
  uint32_t rg_id;   // index of the row group (consumers keep the per-row-group constants while it stays the same)
  uint32_t _pad;
};
static_assert(sizeof(TileHdr) <= kHdrBytes, "tile header fits its slot");

constexpr int RB = 4;  // rows a consumer thread works on at a time (independent chains, amortised uniform branches)

// SMEM: CTA-private table in shared memory (else atomics on the global table).
// SIMPLE: every range leaf is a plain int64 range, no dictionary leaves, every stored aggregate is Sum(int64).
// NK / NA: number of key columns / stored aggregates when the instance is specialised for them (-1: read from the descriptor).
// K8: every key code column of the launch is 8 bits wide.  NOCARRY: the host proved from the chunk statistics that no
// int64 Sum can leave 32 bits inside one CTA (values in [0, 2^32) and rows per CTA x max value < 2^32): plain
// fire-and-forget shared-memory adds, no carry bookkeeping.
template <bool SMEM, bool SIMPLE, int NK, int NA, bool K8, bool NOCARRY>
__global__ void __launch_bounds__(kTaThreads, 1) k_tile_agg(const __grid_constant__ TileAggDesc d) {
  extern __shared__ __align__(128) uint8_t dyn[];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t S = d.n_stages;
  // layout: [full[S] | empty[S]] (8 bytes each, 128 reserved) [headers S x 256] [ring S x slot_bytes] [table]
  const uint32_t bars = smem_u32(dyn);
  uint8_t* const hdrs = dyn + 128;
  uint8_t* const ring = hdrs + S * kHdrBytes;
  uint8_t* const table = ring + size_t(S) * d.slot_bytes;
  const uint32_t ring_s = smem_u32(ring);
  const uint32_t R = 1u << d.rep_log2, n_cells = d.table_slots << d.rep_log2;

  if (tid == 0) {
    for (uint32_t s = 0; s < S; s++) {
      mbar_init(bars + s * 8, 1);                          // full: the producer's expect_tx arrive
      mbar_init(bars + (S + s) * 8, kTaConsumerWarps);     // empty: one arrive per consumer warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (SMEM) {
    uint32_t* c32 = reinterpret_cast<uint32_t*>(table);
    for (uint32_t i = tid; i < n_cells; i += blockDim.x) c32[i] = 0;
    for (uint32_t a = 0; a < d.na; a++) {
      if (d.cell64[a]) {
        const unsigned long long ident = (unsigned long long)agg_identity(uint8_t(d.agg_func[a] & 0xffu), (d.agg_func[a] >> 8) != 0);
        unsigned long long* c = reinterpret_cast<unsigned long long*>(table + d.cell_off[a]);
        for (uint32_t i = tid; i < n_cells; i += blockDim.x) c[i] = ident;
      } else {
        uint32_t* c = reinterpret_cast<uint32_t*>(table + d.cell_off[a]);
        for (uint32_t i = tid; i < n_cells; i += blockDim.x) c[i] = 0;
      }
    }
  }
  __syncthreads();

  const uint32_t CH = d.chunk_tiles, G = gridDim.x, b = blockIdx.x;
  // a CTA takes chunks of CH consecutive tiles, chunk b, b + G, ...; tile, ring stage and phase advance by
  // additions only (no division per tile and thread)
  struct TileIter {
    uint32_t tile, within, st, ph;
  };
  auto iter_begin = [&]() { return TileIter{b * CH, 0u, 0u, 0u}; };
  auto iter_next = [&](TileIter& t) {
    t.tile++;
    if (++t.within == CH) {
      t.within = 0;
      t.tile += (G - 1u) * CH;
    }
    if (++t.st == S) {
      t.st = 0;
      t.ph ^= 1u;
    }
  };

  if (warp == kTaConsumerWarps) {
    // ================================ producer warp ================================
    uint32_t rg = 0, rg_lo = 0, rg_hi = 0, n_rows = 0, rg_cached = 0xffffffffu;
    unsigned long long w0 = 0, w1 = 0;  // this lane's two words of the current row group's descriptor
    static_assert(sizeof(TileAggRg) / 8 <= 64, "descriptor fits two words per lane");
    uint32_t it = 0;
    for (TileIter ti = iter_begin(); ti.tile < d.n_tiles; iter_next(ti), it++) {
      const uint32_t tile = ti.tile, st = ti.st, ph = ti.ph;
      if (tile >= rg_hi) {
        while (tile >= __ldg(d.rg_first_tile + rg + 1)) rg++;
        rg_lo = __ldg(d.rg_first_tile + rg);
        rg_hi = __ldg(d.rg_first_tile + rg + 1);
      }
      if (rg != rg_cached) {
        const unsigned long long* src = reinterpret_cast<const unsigned long long*>(d.rgs + rg);
        w0 = uint32_t(lane) < sizeof(TileAggRg) / 8 ? __ldg(src + lane) : 0ull;
        w1 = uint32_t(lane) + 32u < sizeof(TileAggRg) / 8 ? __ldg(src + lane + 32) : 0ull;
        n_rows = __ldg(&d.rgs[rg].n_rows);
        rg_cached = rg;
      }
      if (it >= S) mbar_wait(bars + (S + st) * 8, ph ^ 1u);  // the consumers are done with the tile that lived here
      const uint32_t r0 = (tile - rg_lo) * d.tile_rows;
      const uint32_t n = min(d.tile_rows, n_rows - r0);
      TileHdr* h = reinterpret_cast<TileHdr*>(hdrs + st * kHdrBytes);
      {
        unsigned long long* dst = reinterpret_cast<unsigned long long*>(&h->rg);
        if (uint32_t(lane) < sizeof(TileAggRg) / 8) dst[lane] = w0;
        if (uint32_t(lane) + 32u < sizeof(TileAggRg) / 8) dst[lane + 32] = w1;
        if (lane == 0) {
          h->r0 = r0;
          h->n = n;
          h->rg_id = rg;
        }
      }
      __syncwarp();
      if (lane == 0) {
        const uint32_t full = bars + st * 8;
        const uint32_t slot = ring_s + st * d.slot_bytes;
        uint32_t bytes = 0;
        uint32_t pb[kTaPlain], cb[kTaCodes];
#pragma unroll
        for (int p = 0; p < kTaPlain; p++) {
          pb[p] = (uint32_t(p) < d.n_plain && h->rg.plain[p] != nullptr) ? ((n * 8u + 15u) & ~15u) : 0u;
          bytes += pb[p];
        }
#pragma unroll
        for (int c = 0; c < kTaCodes; c++) {
          cb[c] = (uint32_t(c) < d.n_codes && h->rg.codes[c] != nullptr) ? ((n * (uint32_t(h->rg.code_w[c]) >> 3) + 15u) & ~15u) : 0u;
          bytes += cb[c];
        }
        mbar_expect_tx(full, bytes);
#pragma unroll
        for (int p = 0; p < kTaPlain; p++)
          if (pb[p]) bulk_g2s(slot + d.plain_off[p], h->rg.plain[p] + size_t(r0) * 8u, pb[p], full);
#pragma unroll
        for (int c = 0; c < kTaCodes; c++)
          if (cb[c]) bulk_g2s(slot + d.code_off[c], h->rg.codes[c] + size_t(r0) * (h->rg.code_w[c] >> 3), cb[c], full);
      }
      __syncwarp();
    }
  } else {
    // ================================ consumer warps ================================
    constexpr bool RTK = NK < 0, RTA = NA < 0;  // key / aggregate counts known at run time only
    uint32_t sel = 0;
    const uint32_t table_s = smem_u32(table);
    const uint32_t rep = uint32_t(lane) & (R - 1u);
    const uint32_t nk = RTK ? d.nk : uint32_t(NK), na = RTA ? d.na : uint32_t(NA);
    // constants of the row group the tiles come from (refreshed when the header names another row group)
    uint32_t cur_rg = 0xffffffffu;
    long long lo[kTaLeaves], hi[kTaLeaves];
    uint32_t loff[kTaLeaves];
    bool leval[kTaLeaves];
    uint32_t poff[kTaPreds], psh[kTaPreds], pbias[kTaPreds];
    const uint8_t* plut[kTaPreds];
    bool peval[kTaPreds];
    bool tile_pass = true;
    // a key column that is absent from the row group (every row NULL) reads any staged byte with stride 0
    uint32_t koff[kTaKeys], ksh[kTaKeys], kbias[kTaKeys], kstride[kTaKeys];
#pragma unroll
    for (int l = 0; l < kTaLeaves; l++) { lo[l] = hi[l] = 0; loff[l] = 0; leval[l] = false; }
#pragma unroll
    for (int p = 0; p < kTaPreds; p++) { poff[p] = psh[p] = pbias[p] = 0; plut[p] = nullptr; peval[p] = false; }
#pragma unroll
    for (int k = 0; k < kTaKeys; k++) { koff[k] = ksh[k] = kbias[k] = kstride[k] = 0; }
    uint32_t aoff[kTaAggs];
#pragma unroll
    for (int a = 0; a < kTaAggs; a++) aoff[a] = uint32_t(a) < na ? d.plain_off[d.agg_plain[a]] : 0u;

    for (TileIter ti = iter_begin(); ti.tile < d.n_tiles; iter_next(ti)) {
      const uint32_t st = ti.st, ph = ti.ph;
      mbar_wait(bars + st * 8, ph);
      const TileHdr* h = reinterpret_cast<const TileHdr*>(hdrs + st * kHdrBytes);
      const uint32_t slot_s = ring_s + st * d.slot_bytes;
      const uint32_t n = h->n;
      if (h->rg_id != cur_rg) {  // warp-uniform
        cur_rg = h->rg_id;
#pragma unroll
        for (int l = 0; l < kTaLeaves; l++) {
          leval[l] = uint32_t(l) < d.nl && !h->rg.leaf_skip[l];
          lo[l] = leval[l] ? h->rg.lo[l] : 0;
          hi[l] = leval[l] ? h->rg.hi[l] : 0;
          loff[l] = leval[l] ? d.plain_off[d.leaf_plain[l]] : 0u;
        }
        tile_pass = true;
        if (!SIMPLE) {
#pragma unroll
          for (int p = 0; p < kTaPreds; p++) {
            plut[p] = uint32_t(p) < d.np ? h->rg.pred_lut[p] : nullptr;
            peval[p] = plut[p] != nullptr;
            if (peval[p]) {
              const uint32_t c = d.pred_code[p];
              if (h->rg.codes[c] == nullptr) {  // column absent: every row NULL
                peval[p] = false;
                tile_pass = tile_pass && d.pred_null[p] != 0;
              } else {
                poff[p] = d.code_off[c];
                psh[p] = uint32_t(h->rg.code_w[c]) >> 4;  // 8 -> 0, 16 -> 1, 32 -> 2
                pbias[p] = h->rg.code_bias[c];
              }
            }
          }
        }
#pragma unroll
        for (int k = 0; k < kTaKeys; k++) {
          if (uint32_t(k) < nk) {
            const uint32_t c = d.key_code[k];
            const bool on = h->rg.codes[c] != nullptr;
            koff[k] = on ? d.code_off[c] : 0u;
            ksh[k] = on ? uint32_t(h->rg.code_w[c]) >> 4 : 0u;
            kbias[k] = on ? uint32_t(h->rg.code_bias[c]) : 0u;
            kstride[k] = on ? d.key_stride[k] : 0u;
          }
        }
      }

      if (tile_pass) {
        for (uint32_t base = uint32_t(tid); base < n; base += RB * NC) {
          uint32_t r[RB];  // row inside the tile (clamped: loads of rows past the end stay inside the staged tile)
          bool act[RB];
#pragma unroll
          for (int j = 0; j < RB; j++) {
            const uint32_t rj = base + uint32_t(j) * NC;
            act[j] = rj < n;
            r[j] = act[j] ? rj : base;
          }
          // ---- range leaves ----
#pragma unroll
          for (int l = 0; l < kTaLeaves; l++) {
            if (leval[l]) {
              const uint32_t cb = slot_s + loff[l];
              if (SIMPLE) {
#pragma unroll
                for (int j = 0; j < RB; j++) {
                  const long long x = (long long)lds64(cb + r[j] * 8u);
                  act[j] = act[j] && x >= lo[l] && x <= hi[l];
                }
              } else {
                const uint32_t f = d.leaf_flags[l];
#pragma unroll
                for (int j = 0; j < RB; j++) {
                  const long long x = (long long)lds64(cb + r[j] * 8u);
                  bool in;
                  if (f & 1u) {
                    const double xd = (f & 2u) ? __longlong_as_double(x) : double(x);
                    in = xd >= __longlong_as_double(lo[l]) && xd <= __longlong_as_double(hi[l]);
                  } else {
                    in = x >= lo[l] && x <= hi[l];
                  }
                  act[j] = act[j] && (in != ((f & 4u) != 0));
                }
              }
            }
          }
          // ---- dictionary leaves: one result byte per dictionary id ----
          if (!SIMPLE) {
#pragma unroll
            for (int p = 0; p < kTaPreds; p++) {
              if (peval[p]) {
                const uint32_t cb = slot_s + poff[p];
#pragma unroll
                for (int j = 0; j < RB; j++) {
                  const uint32_t code = psh[p] == 0 ? lds8(cb + r[j]) : (psh[p] == 1 ? lds16(cb + r[j] * 2u) : lds32(cb + r[j] * 4u));
                  const bool isnull = pbias[p] == 0u && code == 0u;
                  const uint32_t id = isnull ? 0u : code + pbias[p] - 1u;
                  const bool pass = isnull ? (d.pred_null[p] != 0) : (__ldg(plut[p] + id) != 0);
                  act[j] = act[j] && pass;
                }
              }
            }
          }
          // ---- dense slot ----
          uint32_t slot[RB];
#pragma unroll
          for (int j = 0; j < RB; j++) {
            slot[j] = 0;
            sel += act[j] ? 1u : 0u;
          }
#pragma unroll
          for (int k = 0; k < kTaKeys; k++) {
            if (uint32_t(k) < nk) {
              const uint32_t cb = slot_s + koff[k];
              if (K8 || ksh[k] == 0) {
#pragma unroll
                for (int j = 0; j < RB; j++) slot[j] += (lds8(cb + r[j]) + kbias[k]) * kstride[k];
              } else if (ksh[k] == 1) {
#pragma unroll
                for (int j = 0; j < RB; j++) slot[j] += (lds16(cb + r[j] * 2u) + kbias[k]) * kstride[k];
              } else {
#pragma unroll
                for (int j = 0; j < RB; j++) slot[j] += (lds32(cb + r[j] * 4u) + kbias[k]) * kstride[k];
              }
            }
          }
          // ---- fold into the table ----
          if (SMEM) {
#pragma unroll
            for (int j = 0; j < RB; j++) {
              slot[j] = (slot[j] << d.rep_log2) + rep;  // cell index (global slot = cell >> rep_log2)
              red_add_shared_if(table_s + slot[j] * 4u, 1u, act[j]);
            }
#pragma unroll
            for (int a = 0; a < kTaAggs; a++) {
              if (uint32_t(a) < na) {
                const uint32_t cb = slot_s + aoff[a];
                if (SIMPLE || !d.cell64[a]) {
                  const uint32_t cells_s = table_s + d.cell_off[a];
                  if (NOCARRY) {
#pragma unroll
                    for (int j = 0; j < RB; j++) red_add_shared_if(cells_s + slot[j] * 4u, uint32_t(lds64(cb + r[j] * 8u)), act[j]);
                    continue;
                  }
                  uint32_t up[RB], any_up = 0;
#pragma unroll
                  for (int j = 0; j < RB; j++) {
                    const unsigned long long v = lds64(cb + r[j] * 8u);
                    const uint32_t vlo = uint32_t(v);
                    const uint32_t old = atom_add_shared_if(cells_s + slot[j] * 4u, vlo, act[j]);
                    up[j] = act[j] ? uint32_t(v >> 32) + ((old + vlo < old) ? 1u : 0u) : 0u;  // high word + carry out of the low word
                    any_up |= up[j];
                  }
                  if (any_up) {  // values beyond 32 bits / a low word that wrapped: the global cell takes the rest
#pragma unroll
                    for (int j = 0; j < RB; j++)
                      if (up[j]) atomicAdd(reinterpret_cast<unsigned long long*>(d.t_agg[a] + (slot[j] >> d.rep_log2)), (unsigned long long)up[j] << 32);
                  }
                } else {
                  unsigned long long* cells = reinterpret_cast<unsigned long long*>(table + d.cell_off[a]);
                  const uint32_t func = d.agg_func[a] & 0xffu;
                  const bool isf = (d.agg_func[a] >> 8) != 0;
#pragma unroll
                  for (int j = 0; j < RB; j++)
                    if (act[j]) smem_apply64(func, isf, cells + slot[j], (long long)lds64(cb + r[j] * 8u));
                }
              }
            }
          } else {
#pragma unroll
            for (int j = 0; j < RB; j++)
              if (act[j]) atomicAdd(d.t_rows + slot[j], 1ull);
#pragma unroll
            for (int a = 0; a < kTaAggs; a++) {
              if (uint32_t(a) < na) {
                const uint32_t cb = slot_s + aoff[a];
                const uint8_t func = SIMPLE ? uint8_t(1) : uint8_t(d.agg_func[a] & 0xffu);
                const bool isf = SIMPLE ? false : (d.agg_func[a] >> 8) != 0;
#pragma unroll
                for (int j = 0; j < RB; j++)
                  if (act[j]) apply_agg(func, isf, d.t_agg[a] + slot[j], (long long)lds64(cb + r[j] * 8u));
              }
            }
          }
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(bars + (S + st) * 8);
    }
    sel = __reduce_add_sync(FULL, sel);
    if (lane == 0 && sel) atomicAdd(d.counters, (unsigned long long)sel);
  }
  __syncthreads();
  // ================================ epilogue: CTA table -> global table ================================
  if (SMEM) {
    const uint32_t* t_cnt = reinterpret_cast<const uint32_t*>(table);
    // every CTA starts its fold at another slot: the CTAs of a launch finish together, and 148 of them walking the
    // same addresses in the same order serialise in the L2 atomic units
    const uint32_t rot = uint32_t((uint64_t(blockIdx.x) * d.table_slots) / gridDim.x);
    for (uint32_t i = tid; i < d.table_slots; i += blockDim.x) {
      uint32_t s = i + rot;
      if (s >= d.table_slots) s -= d.table_slots;
      unsigned long long c = 0;
      for (uint32_t r = 0; r < R; r++) c += t_cnt[(s << d.rep_log2) + r];
      if (c == 0) continue;
      atomicAdd(d.t_rows + s, c);
      for (uint32_t a = 0; a < d.na; a++) {
        const uint8_t func = uint8_t(d.agg_func[a] & 0xffu);
        const bool isf = (d.agg_func[a] >> 8) != 0;
        if (d.cell64[a]) {
          const long long* cells = reinterpret_cast<const long long*>(table + d.cell_off[a]) + (s << d.rep_log2);
          long long v = cells[0];
          for (uint32_t r = 1; r < R; r++) v = agg_combine(func, isf, v, cells[r]);
          apply_agg(func, isf, d.t_agg[a] + s, v);
        } else {
          const uint32_t* cells = reinterpret_cast<const uint32_t*>(table + d.cell_off[a]) + (s << d.rep_log2);
          unsigned long long v = 0;
          for (uint32_t r = 0; r < R; r++) v += cells[r];
          if (v) atomicAdd(reinterpret_cast<unsigned long long*>(d.t_agg[a] + s), v);
        }
      }
    }
  }
}

}  // namespace

size_t tile_agg_smem_bytes(const TileAggDesc& d) {
  return 128 + size_t(d.n_stages) * kHdrBytes + size_t(d.n_stages) * d.slot_bytes + (d.smem_table ? d.table_bytes : 0);
}

namespace {
using TaKern = void (*)(const TileAggDesc);
template <int NK, bool K8, bool NOCARRY>
TaKern simple_smem_na(int na) {
  switch (na) {
    case 0: return k_tile_agg<true, true, NK, 0, K8, NOCARRY>;
    case 1: return k_tile_agg<true, true, NK, 1, K8, NOCARRY>;
    case 2: return k_tile_agg<true, true, NK, 2, K8, NOCARRY>;
    default: return nullptr;
  }
}
template <bool K8, bool NOCARRY>
TaKern simple_smem_nk(int nk, int na) {
  switch (nk) {
    case 0: return simple_smem_na<0, K8, NOCARRY>(na);
    case 1: return simple_smem_na<1, K8, NOCARRY>(na);
    case 2: return simple_smem_na<2, K8, NOCARRY>(na);
    case 3: return simple_smem_na<3, K8, NOCARRY>(na);
    case 4: return simple_smem_na<4, K8, NOCARRY>(na);
    default: return nullptr;
  }
}
TaKern simple_smem(int nk, int na, bool k8, bool nocarry) {
  if (k8) return nocarry ? simple_smem_nk<true, true>(nk, na) : simple_smem_nk<true, false>(nk, na);
  return nocarry ? simple_smem_nk<false, true>(nk, na) : simple_smem_nk<false, false>(nk, na);
}
}  // namespace

cudaError_t launch_tile_agg(const TileAggDesc& d, int sm_count, cudaStream_t st) {
  if (d.n_tiles == 0) return cudaSuccess;
  const size_t smem = tile_agg_smem_bytes(d);
  bool simple = d.np == 0;
  for (uint32_t l = 0; l < d.nl; l++) simple = simple && d.leaf_flags[l] == 0;
  for (uint32_t a = 0; a < d.na; a++) simple = simple && d.cell64[a] == 0;
  TaKern kern = nullptr;
  if (simple && d.smem_table) kern = simple_smem(int(d.nk), int(d.na), d.keys8 != 0, d.sums_fit32 != 0);
  if (!kern) {
    if (d.smem_table) kern = simple ? k_tile_agg<true, true, -1, -1, false, false> : k_tile_agg<true, false, -1, -1, false, false>;
    else kern = simple ? k_tile_agg<false, true, -1, -1, false, false> : k_tile_agg<false, false, -1, -1, false, false>;
  }
  const cudaError_t e = kernel_smem_at_least(reinterpret_cast<const void*>(kern), smem);
  if (e != cudaSuccess) return e;
  uint32_t grid = uint32_t(sm_count);
  const uint32_t need = (d.n_tiles + d.chunk_tiles - 1) / d.chunk_tiles;
  if (grid > need) grid = need;
  kern<<<grid, kTaThreads, smem, st>>>(d);
  return cudaGetLastError();
}

}  // namespace fgpu
