// k_take_*: filter-only plans (TableScan -> Filter -> Projection(columns)) over PLAIN int64/double columns.
//
// Takes over PredicateFilter.Callback's filter() (physicalplan/filter.go:276-323: bitmap -> index ranges ->
// per-column Slice + Concatenate, i.e. an ORDER-PRESERVING compaction of every projected column) for the
// plan shape of BASELINE config 5: a conjunction of <= 2 int64 range leaves on PLAIN non-null columns and <= 2
// dictionary-column leaves (==, !=, contains, regex, == NULL: one result byte per dictionary id, the column read as a
// flat code array, k_flatten) — any of them possibly decided by the chunk statistics — and <= 4 projected PLAIN
// non-null int64/double columns.  Everything else (projected dictionary columns, NULL values, OR / nested leaves)
// stays with k_rows in kernels.cu.
//
// Two passes over spans (the contiguous piece of a row group a warp takes per turn, in scan order):
//   k_take_count  reads only the leaf columns and leaves the number of passing rows of every span;
//   k_take_scan   turns the counts into output bases (one CTA, exclusive scan);
//   k_take_write  re-evaluates the leaves and writes the projected values of the passing rows at
//                 base + rank (rank from warp votes), reading the projected columns only where a row
//                 passed.  Spans of row groups whose leaves were all decided by statistics are plain copies.
// No shared memory: every lane keeps 8 independent 8-byte loads in flight per leaf column (a 256-row block
// per warp and step), the loads of a warp are 256 contiguous bytes.
//
// Algorithmic bytes per row: 8 per leaf column that must be evaluated (read twice: traffic 16) + per
// selected row 8 read + 8 written per projected column.
#include <cuda_runtime.h>

#include "device_types.h"
#include "kernels.h"

namespace fgpu {
namespace {

constexpr unsigned FULL = 0xffffffffu;
constexpr int kTakeThreads = 256;
constexpr int kTakeWarps = kTakeThreads / 32;
constexpr uint32_t kBlockRows = 256;  // rows a warp handles per iteration (8 steps of 32)

struct SpanPos {
  const TakeRg* R;
  uint32_t row0, row_end;
};

__device__ __forceinline__ SpanPos locate(const TakeDesc& d, uint32_t span, uint32_t& rg) {
  while (span >= __ldg(d.rg_first_span + rg + 1)) rg++;
  SpanPos p;
  p.R = d.rgs + rg;
  const uint32_t span_rows = d.span_blocks * kBlockRows;
  p.row0 = (span - __ldg(d.rg_first_span + rg)) * span_rows;
  p.row_end = min(__ldg(&p.R->n_rows), p.row0 + span_rows);
  return p;
}

struct Preds {  // the dictionary leaves of one row group
  const uint8_t* codes[kTakePreds];
  const uint8_t* lut[kTakePreds];
  uint32_t w[kTakePreds], bias[kTakePreds], pnull[kTakePreds];
};
__device__ __forceinline__ Preds load_preds(const TakeRg* R) {
  Preds P;
#pragma unroll
  for (int p = 0; p < kTakePreds; p++) {
    P.codes[p] = reinterpret_cast<const uint8_t*>(__ldg(reinterpret_cast<const unsigned long long*>(&R->pred_codes[p])));
    P.lut[p] = reinterpret_cast<const uint8_t*>(__ldg(reinterpret_cast<const unsigned long long*>(&R->pred_lut[p])));
    P.w[p] = __ldg(&R->pred_w[p]);
    P.bias[p] = __ldg(&R->pred_bias[p]);
    P.pnull[p] = __ldg(&R->pred_null[p]);
  }
  return P;
}

// pass mask of the 8 steps of one block for this lane (bit j: row r0 + 32 j + lane passes every leaf)
template <int NL, bool HP>
__device__ __forceinline__ uint32_t block_mask(const long long* (&col)[NL > 0 ? NL : 1], const long long (&lo)[NL > 0 ? NL : 1],
                                               const long long (&hi)[NL > 0 ? NL : 1], const Preds& P, uint32_t r0, uint32_t row_end, int lane) {
  uint32_t m = 0;
#pragma unroll
  for (int j = 0; j < 8; j++)
    if (r0 + uint32_t(j) * 32u + uint32_t(lane) < row_end) m |= 1u << j;
#pragma unroll
  for (int l = 0; l < NL; l++) {
    if (col[l] == nullptr) continue;  // decided by the chunk statistics
    long long x[8];
#pragma unroll
    for (int j = 0; j < 8; j++) x[j] = ((m >> j) & 1u) ? __ldg(col[l] + r0 + uint32_t(j) * 32u + uint32_t(lane)) : 0;
#pragma unroll
    for (int j = 0; j < 8; j++)
      if (!(x[j] >= lo[l] && x[j] <= hi[l])) m &= ~(1u << j);
  }
  if constexpr (HP) {
#pragma unroll
    for (int p = 0; p < kTakePreds; p++) {
      if (P.codes[p] == nullptr) continue;
      uint32_t code[8];
#pragma unroll
      for (int j = 0; j < 8; j++) {
        const size_t r = size_t(r0) + uint32_t(j) * 32u + uint32_t(lane);
        code[j] = 0;
        if ((m >> j) & 1u)
          code[j] = P.w[p] == 8 ? uint32_t(__ldg(P.codes[p] + r))
                                : (P.w[p] == 16 ? uint32_t(__ldg(reinterpret_cast<const uint16_t*>(P.codes[p]) + r)) : __ldg(reinterpret_cast<const uint32_t*>(P.codes[p]) + r));
      }
#pragma unroll
      for (int j = 0; j < 8; j++) {
        if (!((m >> j) & 1u)) continue;
        const bool isnull = P.bias[p] == 0u && code[j] == 0u;
        const bool pass = isnull ? (P.pnull[p] != 0u) : (__ldg(P.lut[p] + (code[j] + P.bias[p] - 1u)) != 0);
        if (!pass) m &= ~(1u << j);
      }
    }
  }
  return m;
}

template <int NL, bool HP>
__global__ void __launch_bounds__(kTakeThreads) k_take_count(const __grid_constant__ TakeDesc d) {
  const int lane = threadIdx.x & 31;
  const uint32_t gw = blockIdx.x * kTakeWarps + (threadIdx.x >> 5), GW = gridDim.x * kTakeWarps;
  uint32_t rg = 0;
  for (uint32_t span = gw; span < d.n_spans; span += GW) {
    const SpanPos p = locate(d, span, rg);
    uint32_t cnt = 0;
    if ((NL == 0 && !HP) || __ldg(&p.R->all_pass)) {
      if (lane == 0) d.span_count[span] = p.row_end - p.row0;
      continue;
    }
    const long long* col[NL > 0 ? NL : 1];
    long long lo[NL > 0 ? NL : 1], hi[NL > 0 ? NL : 1];
#pragma unroll
    for (int l = 0; l < NL; l++) {
      col[l] = reinterpret_cast<const long long*>(__ldg(reinterpret_cast<const unsigned long long*>(&p.R->leaf_col[l])));
      lo[l] = __ldg(&p.R->lo[l]);
      hi[l] = __ldg(&p.R->hi[l]);
    }
    Preds P{};
    if (HP) P = load_preds(p.R);
    for (uint32_t r0 = p.row0; r0 < p.row_end; r0 += kBlockRows) cnt += __popc(block_mask<NL, HP>(col, lo, hi, P, r0, p.row_end, lane));
    cnt = __reduce_add_sync(FULL, cnt);
    if (lane == 0) d.span_count[span] = cnt;
  }
}

// span_count[i] := sum of span_count[0..i) (in place, n + 1 entries; one CTA)
__global__ void __launch_bounds__(1024) k_take_scan(unsigned long long* counts, uint32_t n, unsigned long long* total_out) {
  __shared__ unsigned long long warp_sums[32];
  __shared__ unsigned long long carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (uint32_t base = 0; base < n; base += 1024) {
    const uint32_t i = base + threadIdx.x;
    const unsigned long long v = i < n ? counts[i] : 0;
    unsigned long long x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      unsigned long long y = __shfl_up_sync(FULL, x, o);
      if (lane >= o) x += y;
    }
    if (lane == 31) warp_sums[warp] = x;
    __syncthreads();
    if (warp == 0) {
      unsigned long long w = warp_sums[lane], ws = w;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        unsigned long long y = __shfl_up_sync(FULL, ws, o);
        if (lane >= o) ws += y;
      }
      warp_sums[lane] = ws - w;  // exclusive
    }
    __syncthreads();
    const unsigned long long excl = carry + warp_sums[warp] + x - v;
    if (i < n) counts[i] = excl;
    __syncthreads();
    if (threadIdx.x == 1023) carry = excl + v;
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    counts[n] = carry;
    *total_out = carry;
  }
}

template <int NL, int NO, bool HP>
__global__ void __launch_bounds__(kTakeThreads) k_take_write(const __grid_constant__ TakeDesc d) {
  const int lane = threadIdx.x & 31;
  const uint32_t lt = (1u << lane) - 1u;
  const uint32_t gw = blockIdx.x * kTakeWarps + (threadIdx.x >> 5), GW = gridDim.x * kTakeWarps;
  uint32_t rg = 0;
  for (uint32_t span = gw; span < d.n_spans; span += GW) {
    const SpanPos p = locate(d, span, rg);
    unsigned long long base = d.span_count[span];  // exclusive prefix: first output row of this span
    if (d.span_count[span + 1] == base) continue;  // nothing passes here
    const long long* out_col[NO];
#pragma unroll
    for (int o = 0; o < NO; o++) out_col[o] = reinterpret_cast<const long long*>(__ldg(reinterpret_cast<const unsigned long long*>(&p.R->out_col[o])));
    if ((NL == 0 && !HP) || __ldg(&p.R->all_pass)) {  // plain copy of the span
      for (uint32_t r = p.row0 + uint32_t(lane); r < p.row_end; r += 32u) {
#pragma unroll
        for (int o = 0; o < NO; o++) d.out_data[o][base + (r - p.row0)] = __ldg(out_col[o] + r);
      }
      continue;
    }
    const long long* col[NL > 0 ? NL : 1];
    long long lo[NL > 0 ? NL : 1], hi[NL > 0 ? NL : 1];
#pragma unroll
    for (int l = 0; l < NL; l++) {
      col[l] = reinterpret_cast<const long long*>(__ldg(reinterpret_cast<const unsigned long long*>(&p.R->leaf_col[l])));
      lo[l] = __ldg(&p.R->lo[l]);
      hi[l] = __ldg(&p.R->hi[l]);
    }
    Preds P{};
    if (HP) P = load_preds(p.R);
    for (uint32_t r0 = p.row0; r0 < p.row_end; r0 += kBlockRows) {
      const uint32_t m = block_mask<NL, HP>(col, lo, hi, P, r0, p.row_end, lane);
      if (__ballot_sync(FULL, m != 0) == 0) continue;
#pragma unroll
      for (int j = 0; j < 8; j++) {
        const bool pass = (m >> j) & 1u;
        const unsigned vote = __ballot_sync(FULL, pass);
        if (pass) {
          const unsigned long long at = base + __popc(vote & lt);
          const uint32_t r = r0 + uint32_t(j) * 32u + uint32_t(lane);
#pragma unroll
          for (int o = 0; o < NO; o++) d.out_data[o][at] = __ldg(out_col[o] + r);
        }
        base += __popc(vote);
      }
    }
  }
}

template <typename K>
cudaError_t run(K kern, const TakeDesc& d, int sm_count, cudaStream_t st) {
  int per_sm = 0;
  const cudaError_t e = kernel_ctas_per_sm(reinterpret_cast<const void*>(kern), kTakeThreads, 0, &per_sm);
  if (e != cudaSuccess) return e;
  uint32_t grid = uint32_t(sm_count) * uint32_t(per_sm);
  const uint32_t need = (d.n_spans + kTakeWarps - 1) / kTakeWarps;
  if (grid > need) grid = need;
  kern<<<grid, kTakeThreads, 0, st>>>(d);
  return cudaGetLastError();
}

template <int NL, bool HP>
cudaError_t write_no(const TakeDesc& d, int sm_count, cudaStream_t st) {
  switch (d.n_out) {
    case 1: return run(k_take_write<NL, 1, HP>, d, sm_count, st);
    case 2: return run(k_take_write<NL, 2, HP>, d, sm_count, st);
    case 3: return run(k_take_write<NL, 3, HP>, d, sm_count, st);
    default: return run(k_take_write<NL, 4, HP>, d, sm_count, st);
  }
}

template <bool HP>
cudaError_t take_hp(const TakeDesc& d, int sm_count, cudaStream_t st) {
  cudaError_t e;
  switch (d.nl) {
    case 0: e = run(k_take_count<0, HP>, d, sm_count, st); break;
    case 1: e = run(k_take_count<1, HP>, d, sm_count, st); break;
    default: e = run(k_take_count<2, HP>, d, sm_count, st); break;
  }
  if (e != cudaSuccess) return e;
  k_take_scan<<<1, 1024, 0, st>>>(d.span_count, d.n_spans, d.total);
  e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  switch (d.nl) {
    case 0: return write_no<0, HP>(d, sm_count, st);
    case 1: return write_no<1, HP>(d, sm_count, st);
    default: return write_no<2, HP>(d, sm_count, st);
  }
}

}  // namespace

int take_resident_warps(int sm_count) { return sm_count * 8 * kTakeWarps; }  // sizing hint for the host (spans per warp)

cudaError_t launch_take(const TakeDesc& d, int sm_count, cudaStream_t st) {
  if (d.n_spans == 0) return cudaSuccess;
  return d.np ? take_hp<true>(d, sm_count, st) : take_hp<false>(d, sm_count, st);
}

}  // namespace fgpu
