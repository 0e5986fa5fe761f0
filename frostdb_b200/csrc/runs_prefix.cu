// k_runs_prefix: group-by Sum / Count for the ALL-PASS row groups of sorted parts (sm_90a).  The plan shape is the one of
// k_runs_tma (runs_tma.cu), restricted to row groups whose filter the chunk statistics decided (every row passes), with
// no undecided dictionary leaf and only Sum(int64) as stored aggregates.  Such a row group holds a few thousand runs of
// one group each; instead of streaming the rows, the rows [b, e) of one SEGMENT (a maximal stretch with one dense slot)
// add e - b and, for every Sum input, P[e] - P[b] from its exclusive prefix sum (ensure_narrow: P[i] = v[0] + ... +
// v[i-1] modulo 2^64) — exactly the wrapping int64 sum.
//
// The segments depend only on the key columns' run directories and the dense strides, so they are found once per
// compiled plan (k_prefix_segs) and kept grouped by slot (CSR: seg_off, seg).  Work unit of that build: a WINDOW of
// rows of one row group (cut by the host, about 32 run starts each), one warp per window.  The warp finds the run of
// every key column that holds the window's first and last row (128-row seed + a ballot walk), then its lanes take the
// window's SEGMENT BOUNDARIES in parallel: the window start and every run start of every key column inside the window,
// a start shared by several columns kept only for the first of them.  A lane finds the runs of the other columns that
// hold its boundary by binary search in their directory slices (a few L1-resident entries), so the segment's end is
// the nearest next run start of any column (or the window end) and its dense slot the sum of (id + 1) * stride.  The
// build runs twice: count per slot, exclusive scan, scatter.
//
// Every Execute (k_runs_prefix) then gives each slot a group of lanes that folds the slot's list and STORES the
// slot's rows and Sums, 0 for a slot without segments: no atomics, and the launch replaces k_table_init.
#include <cuda_runtime.h>

#include <algorithm>

#include <cub/device/device_scan.cuh>

#include "device_types.h"
#include "kernels.h"
#include "ptx.cuh"

namespace fgpu {
namespace {

constexpr unsigned FULL = 0xffffffffu;
constexpr int kPfWarps = 8;  // warps per CTA (independent)

// Warp-cooperative: index of the run that holds `row` (the last entry whose start <= row), from the row's 128-row seed.
__device__ __forceinline__ uint32_t run_of_row(const Run* runs, const Seed* seeds, uint32_t n_runs, uint32_t row, uint32_t lane) {
  uint32_t k = __ldg(&seeds[row / uint32_t(kIndexRows)].k);
  for (;;) {  // starts increase: the entries behind k that start at or before row form a prefix
    const uint32_t j = k + 1u + lane;
    const uint32_t c = __popc(__ballot_sync(FULL, j < n_runs && __ldg(&runs[j].start) <= row));
    k += c;
    if (c < 32u) return k;
  }
}

// Per lane: the last entry in [lo, hi] whose start <= b (runs[lo].start <= b).
__device__ __forceinline__ uint32_t run_search(const Run* runs, uint32_t lo, uint32_t hi, uint32_t b) {
  while (lo < hi) {
    const uint32_t mid = (lo + hi + 1u) >> 1;
    if (__ldg(&runs[mid].start) <= b) lo = mid;
    else hi = mid - 1u;
  }
  return lo;
}

// kScatter = false: count the segments of every slot; true: write them (cnt counts down to 0 again).
template <bool kScatter>
__global__ void __launch_bounds__(kPfWarps * 32) k_prefix_segs(const __grid_constant__ PrefixBuildDesc d) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t nk = d.nk;
  for (uint32_t w = blockIdx.x * kPfWarps + (threadIdx.x >> 5); w < d.n_win; w += gridDim.x * kPfWarps) {
    const uint4 win = __ldg(reinterpret_cast<const uint4*>(d.wins + w));  // PrefixWin {rg, r0, rows, -}
    const PrefixRg* const R = d.rgs + win.x;
    const uint32_t r0 = win.y, r1 = win.y + win.z;
    const Run* runs[kRunsKeys];
    uint32_t k0[kRunsKeys], k1[kRunsKeys];
    uint32_t nb = 1;  // boundaries: r0, then the starts of runs k0 + 1 .. k1 of every key column
#pragma unroll
    for (int q = 0; q < kRunsKeys; q++) {
      runs[q] = nullptr;
      k0[q] = k1[q] = 0;
      if (uint32_t(q) < nk) {
        runs[q] = ldg_ptr(&R->runs[q]);
        const Seed* seeds = ldg_ptr(&R->seeds[q]);
        const uint32_t n_runs = __ldg(&R->n_runs[q]);
        k0[q] = run_of_row(runs[q], seeds, n_runs, r0, lane);
        k1[q] = run_of_row(runs[q], seeds, n_runs, r1 - 1u, lane);
        nb += k1[q] - k0[q];
      }
    }
    for (uint32_t i = lane; i < nb; i += 32u) {
      // boundary i: 0 is r0; then the run starts of column 0, column 1, ...
      int qb = -1;
      uint32_t kb = 0, rest = i - 1u;
#pragma unroll
      for (int q = 0; q < kRunsKeys; q++) {
        if (i == 0 || qb >= 0 || uint32_t(q) >= nk) continue;
        const uint32_t n = k1[q] - k0[q];
        if (rest < n) {
          qb = q;
          kb = k0[q] + 1u + rest;
        } else {
          rest -= n;
        }
      }
      uint32_t b = r0;
#pragma unroll
      for (int q = 0; q < kRunsKeys; q++)  // (static indices: the pointers stay in registers)
        if (q == qb) b = __ldg(&runs[q][kb].start);
      uint32_t end = r1, slot = 0;
      bool dup = false;
#pragma unroll
      for (int q = 0; q < kRunsKeys; q++) {
        if (uint32_t(q) >= nk) continue;
        const uint32_t k = q == qb ? kb : (qb < 0 ? k0[q] : run_search(runs[q], k0[q], k1[q], b));
        const Run* const e = runs[q] + k;
        if (q < qb && __ldg(&e->start) == b) dup = true;  // column q starts a run here too: its lane takes the boundary
        slot += (__ldg(&e->val) + 1u) * d.stride[q];      // NULL (0xffffffff) contributes 0
        end = min(end, __ldg(&e[1].start));
      }
      if (dup) continue;
      if (kScatter) {
        const uint32_t pos = atomicSub(d.cnt + slot, 1u) - 1u;
        d.seg[__ldg(d.seg_off + slot) + pos] = PrefixSeg{win.x, b, end};
      } else {
        atomicAdd(d.cnt + slot, 1u);
      }
    }
  }
}

constexpr int kPfUnroll = 8;  // segments of one lane in flight

// Lanes sub, sub + G, ... of a slot's list [lo, hi): rows and wrapping Sums, kPfUnroll segments in flight per lane.
__device__ __forceinline__ void fold_list(const PrefixDesc& d, uint32_t lo, uint32_t hi, uint32_t sub, uint32_t G,
                                          unsigned long long& rows, unsigned long long (&agg)[kRunsAggs]) {
  const uint32_t na = d.na;
  for (uint32_t i = lo + sub; i < hi; i += G * kPfUnroll) {
    uint32_t rg[kPfUnroll], b[kPfUnroll], e[kPfUnroll];
#pragma unroll
    for (int u = 0; u < kPfUnroll; u++) {
      const uint32_t j = i + uint32_t(u) * G;
      rg[u] = b[u] = e[u] = 0;
      if (j < hi) {
        const PrefixSeg* sg = d.seg + j;
        rg[u] = __ldg(&sg->rg);
        b[u] = __ldg(&sg->b);
        e[u] = __ldg(&sg->e);
      }
    }
#pragma unroll
    for (int u = 0; u < kPfUnroll; u++) {
      if (e[u] == b[u]) continue;  // past the list (segments are never empty)
      rows += e[u] - b[u];
#pragma unroll
      for (int a = 0; a < kRunsAggs; a++)
        if (uint32_t(a) < na) {
          const long long* pre = ldg_ptr(&d.rgs[rg[u]].pre[a]);
          agg[a] += (unsigned long long)__ldg(pre + e[u]) - (unsigned long long)__ldg(pre + b[u]);
        }
    }
  }
}

__device__ __forceinline__ void store_slot(const PrefixDesc& d, uint32_t slot, unsigned long long rows, const unsigned long long (&agg)[kRunsAggs]) {
  d.t_rows[slot] = rows;
#pragma unroll
  for (int a = 0; a < kRunsAggs; a++)
    if (uint32_t(a) < d.na) d.t_agg[a][slot] = (long long)agg[a];
}

// kCta = false: a group of 1 << group_log2 lanes (<= 32) per slot; true: a CTA per slot (long lists, e.g. a key that
// is not a sort prefix, whose slot collects a segment from every run of every row group).
template <bool kCta>
__global__ void __launch_bounds__(kPfWarps * 32) k_runs_prefix(const __grid_constant__ PrefixDesc d) {
  const uint32_t lane = threadIdx.x & 31u;
  if (blockIdx.x == 0 && threadIdx.x < 10)  // counters + the group counter behind them, as k_table_init leaves them
    d.counters[threadIdx.x] = threadIdx.x == 0 ? d.all_rows : 0ull;  // rows that passed the filter (all of them)
  if (kCta) {
    __shared__ unsigned long long part[kPfWarps][1 + kRunsAggs];
    const uint32_t warp = threadIdx.x >> 5;
    for (uint32_t slot = blockIdx.x; slot < d.n_slots; slot += gridDim.x) {  // (CTA-uniform)
      unsigned long long rows = 0, agg[kRunsAggs] = {0, 0, 0};
      fold_list(d, __ldg(d.seg_off + slot), __ldg(d.seg_off + slot + 1), threadIdx.x, blockDim.x, rows, agg);
      for (int o = 16; o; o >>= 1) {
        rows += __shfl_xor_sync(FULL, rows, o);
#pragma unroll
        for (int a = 0; a < kRunsAggs; a++) agg[a] += __shfl_xor_sync(FULL, agg[a], o);
      }
      if (lane == 0) {
        part[warp][0] = rows;
#pragma unroll
        for (int a = 0; a < kRunsAggs; a++) part[warp][1 + a] = agg[a];
      }
      __syncthreads();
      if (threadIdx.x == 0) {
        for (int w = 1; w < kPfWarps; w++) {
          rows += part[w][0];
#pragma unroll
          for (int a = 0; a < kRunsAggs; a++) agg[a] += part[w][1 + a];
        }
        store_slot(d, slot, rows, agg);
      }
      __syncthreads();
    }
    return;
  }
  const uint32_t g_log2 = d.group_log2, G = 1u << g_log2, sub = lane & (G - 1u);
  const uint32_t per_warp = 32u >> g_log2;
  const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, n_warps = (gridDim.x * blockDim.x) >> 5;
  // (the slot loop is warp-uniform: every lane reaches the shuffles below)
  for (uint32_t base = warp * per_warp; base < d.n_slots; base += n_warps * per_warp) {
    const uint32_t slot = base + (lane >> g_log2);
    uint32_t lo = 0, hi = 0;
    if (slot < d.n_slots) {
      lo = __ldg(d.seg_off + slot);
      hi = __ldg(d.seg_off + slot + 1);
    }
    unsigned long long rows = 0, agg[kRunsAggs] = {0, 0, 0};
    fold_list(d, lo, hi, sub, G, rows, agg);
    for (uint32_t o = G >> 1; o; o >>= 1) {
      rows += __shfl_xor_sync(FULL, rows, o);
#pragma unroll
      for (int a = 0; a < kRunsAggs; a++) agg[a] += __shfl_xor_sync(FULL, agg[a], o);
    }
    if (slot < d.n_slots && sub == 0) store_slot(d, slot, rows, agg);
  }
}

}  // namespace

// Rows per window of a row group whose key directories hold sum_runs entries in all: about 32 run starts per window,
// one per lane (a multiple of kIndexRows, at least 1024 rows); one window when there are no keys.
uint32_t runs_prefix_window_rows(uint32_t n_rows, uint32_t sum_runs) {
  if (sum_runs == 0) return std::max<uint32_t>(n_rows, 1u);
  const uint64_t t = (uint64_t(32) * n_rows / sum_runs) & ~uint64_t(kIndexRows - 1);
  return uint32_t(std::min<uint64_t>(std::max<uint64_t>(t, 1024), std::max<uint32_t>(n_rows, 1u)));
}

namespace {
uint32_t prefix_grid(uint32_t warps, int sm_count) {
  const uint32_t grid = std::max<uint32_t>((warps + kPfWarps - 1) / kPfWarps, 1u);
  return std::min<uint32_t>(grid, uint32_t(sm_count) * (2048u / (kPfWarps * 32u)));
}
size_t scan_temp_bytes(uint32_t n_slots) {
  size_t t = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, t, static_cast<const uint32_t*>(nullptr), static_cast<uint32_t*>(nullptr), int(n_slots + 1));
  return t;
}
}  // namespace

// [cnt: n_slots + 1 counters | 16-byte aligned CUB scan storage]
size_t prefix_build_scratch_bytes(uint32_t n_slots) { return ((size_t(n_slots + 1) * 4 + 15) & ~size_t(15)) + scan_temp_bytes(n_slots); }

cudaError_t launch_prefix_build(PrefixBuildDesc d, uint32_t n_slots, uint32_t* seg_off, void* scratch, int sm_count, cudaStream_t st) {
  d.cnt = static_cast<uint32_t*>(scratch);
  d.seg_off = seg_off;
  const size_t cnt_bytes = (size_t(n_slots + 1) * 4 + 15) & ~size_t(15);
  size_t temp = scan_temp_bytes(n_slots);
  cudaError_t e = cudaMemsetAsync(d.cnt, 0, size_t(n_slots + 1) * 4, st);
  if (e != cudaSuccess) return e;
  const uint32_t grid = prefix_grid(d.n_win, sm_count);
  if (d.n_win) k_prefix_segs<false><<<grid, kPfWarps * 32, 0, st>>>(d);
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  e = cub::DeviceScan::ExclusiveSum(static_cast<uint8_t*>(scratch) + cnt_bytes, temp, d.cnt, seg_off, int(n_slots + 1), st);
  if (e != cudaSuccess) return e;
  if (d.n_win) k_prefix_segs<true><<<grid, kPfWarps * 32, 0, st>>>(d);
  return cudaGetLastError();
}

cudaError_t launch_runs_prefix(const PrefixDesc& d, int sm_count, cudaStream_t st) {
  if (d.group_log2 > 5) {
    k_runs_prefix<true><<<prefix_grid(d.n_slots * kPfWarps, sm_count), kPfWarps * 32, 0, st>>>(d);
  } else {
    const uint32_t per_warp = 32u >> d.group_log2;
    k_runs_prefix<false><<<prefix_grid((d.n_slots + per_warp - 1) / per_warp, sm_count), kPfWarps * 32, 0, st>>>(d);
  }
  return cudaGetLastError();
}

}  // namespace fgpu
