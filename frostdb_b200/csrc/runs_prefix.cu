// k_runs_prefix: group-by Sum / Count for the ALL-PASS row groups of sorted parts (sm_90a).  The plan shape is the one of
// k_runs_tma (runs_tma.cu), restricted to row groups whose filter the chunk statistics decided (every row passes), with
// no undecided dictionary leaf and only Sum(int64) as stored aggregates.  Such a row group holds a few thousand runs of
// one group each; instead of streaming the rows, the kernel reads per group run
//   * the run directories of the key columns (16 B per run, row space, NULL = 0xffffffff contributes 0), and
//   * two entries of the exclusive prefix sum P of every Sum input (ensure_narrow: P[i] = v[0] + ... + v[i-1] modulo
//     2^64), so that the rows [b, e) add P[e] - P[b] — exactly the wrapping int64 sum — and e - b to their group.
//
// Work unit: a WINDOW of rows of one row group (cut by the host, about 32 run starts each), one warp per window.  The
// warp finds the run of every key column that holds the window's first and last row (128-row seed + a ballot walk), then
// its lanes take the window's SEGMENT BOUNDARIES in parallel: the window start and every run start of every key column
// inside the window, a start shared by several columns kept only for the first of them.  A lane finds the runs of the
// other columns that hold its boundary by binary search in their directory slices (a few L1-resident entries), so the
// segment's end is the nearest next run start of any column (or the window end) and its dense slot the sum of
// (id + 1) * stride.  One atomic per segment and table column; adjacent segments have different slots.
#include <cuda_runtime.h>

#include <algorithm>

#include "device_types.h"
#include "kernels.h"

namespace fgpu {
namespace {

constexpr unsigned FULL = 0xffffffffu;
constexpr int kPfWarps = 8;  // warps per CTA (independent)

template <typename T>
__device__ __forceinline__ T ldg_ptr(T const* p) {
  return reinterpret_cast<T>(__ldg(reinterpret_cast<const unsigned long long*>(p)));
}

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

__global__ void __launch_bounds__(kPfWarps * 32) k_runs_prefix(const __grid_constant__ PrefixDesc d) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t nk = d.nk, na = d.na;
  unsigned long long sel = 0;
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
    const long long* pre[kRunsAggs];
#pragma unroll
    for (int a = 0; a < kRunsAggs; a++) pre[a] = uint32_t(a) < na ? ldg_ptr(&R->pre[a]) : nullptr;
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
      atomicAdd(d.t_rows + slot, (unsigned long long)(end - b));
#pragma unroll
      for (int a = 0; a < kRunsAggs; a++)
        if (uint32_t(a) < na)
          atomicAdd(reinterpret_cast<unsigned long long*>(d.t_agg[a]) + slot,
                    (unsigned long long)__ldg(pre[a] + end) - (unsigned long long)__ldg(pre[a] + b));
      sel += end - b;
    }
  }
  for (int o = 16; o; o >>= 1) sel += __shfl_xor_sync(FULL, sel, o);
  if (lane == 0 && sel) atomicAdd(d.counters, sel);  // rows that passed the filter (all of them)
}

}  // namespace

// Rows per window of a row group whose key directories hold sum_runs entries in all: about 32 run starts per window,
// one per lane (a multiple of kIndexRows, at least 1024 rows); one window when there are no keys.
uint32_t runs_prefix_window_rows(uint32_t n_rows, uint32_t sum_runs) {
  if (sum_runs == 0) return std::max<uint32_t>(n_rows, 1u);
  const uint64_t t = (uint64_t(32) * n_rows / sum_runs) & ~uint64_t(kIndexRows - 1);
  return uint32_t(std::min<uint64_t>(std::max<uint64_t>(t, 1024), std::max<uint32_t>(n_rows, 1u)));
}

cudaError_t launch_runs_prefix(const PrefixDesc& d, int sm_count, cudaStream_t st) {
  if (d.n_win == 0) return cudaSuccess;
  uint32_t grid = (d.n_win + kPfWarps - 1) / kPfWarps;
  grid = std::min<uint32_t>(grid, uint32_t(sm_count) * (2048u / (kPfWarps * 32u)));
  k_runs_prefix<<<grid, kPfWarps * 32, 0, st>>>(d);
  return cudaGetLastError();
}

}  // namespace fgpu
