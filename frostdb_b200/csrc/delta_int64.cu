// DELTA_BINARY_PACKED int64 pages of Parquet parts decoded at upload into the dense value array (sm_90a).  The host's
// page walk has validated every stream and listed its miniblocks; the streams sit in the upload's staging buffer.
// A page's values are the inclusive prefix sum, modulo 2^64, of its first value followed by one element per value
// 1 .. n - 1 (the miniblock's min delta plus the packed delta), so the decode is a segmented scan over the upload's
// values, reset at every page start, in three launches whatever the number of pages:
//   k_dbp_local  one warp per 32-value group of a page (a CTA: 32 consecutive groups of the upload).  Each lane unpacks
//                its element with a 64-bit funnel shift from two aligned words, the warp runs an inclusive shuffle
//                scan and writes the local prefixes into the page's hole.  Warp 0 then scans the CTA's 32 group totals,
//                segmented at page starts, and leaves per group its carry from the groups before it in the CTA, per CTA
//                its total since its last page start and whether a page starts in it.
//   k_dbp_carry  one CTA: the segmented exclusive scan of the CTA totals, 1 024 at a time, which gives every CTA the
//                carry of the CTAs before it (up to the last page start).
//   k_dbp_add    one warp per group: adds the group's carry (its CTA's too when its page started in an earlier CTA)
//                to its values.
#include <cuda_runtime.h>

#include "device_types.h"
#include "kernels.h"

namespace fgpu {
namespace {

constexpr unsigned FULL = 0xffffffffu;
constexpr int kThreads = 32 * kDbpGroupsPerCta;

struct Scratch {
  unsigned long long* grp_carry;  // per group: carry from the groups before it in its CTA, since its page start
  uint32_t* grp_page;             // per group: its page
  unsigned long long* cta_sum;    // per CTA: its total since its last page start; k_dbp_carry: its carry-in
  uint32_t* cta_reset;            // per CTA: a page starts in it
};

__host__ __device__ inline size_t al16(size_t n) { return (n + 15) & ~size_t(15); }

__host__ __device__ inline Scratch scratch_of(void* p, uint32_t n_groups) {
  const uint32_t n_ctas = (n_groups + kDbpGroupsPerCta - 1) / kDbpGroupsPerCta;
  uint8_t* b = static_cast<uint8_t*>(p);
  Scratch s;
  s.grp_carry = reinterpret_cast<unsigned long long*>(b);
  b += al16(size_t(n_groups) * 8);
  s.cta_sum = reinterpret_cast<unsigned long long*>(b);
  b += al16(size_t(n_ctas) * 8);
  s.grp_page = reinterpret_cast<uint32_t*>(b);
  b += al16(size_t(n_groups) * 4);
  s.cta_reset = reinterpret_cast<uint32_t*>(b);
  return s;
}

// the page holding group g: the last page whose first group is <= g
__device__ __forceinline__ uint32_t page_of(const DbpPage* pages, uint32_t n_pages, uint32_t g) {
  uint32_t lo = 0, hi = n_pages;
  while (hi - lo > 1) {
    const uint32_t mid = (lo + hi) >> 1;
    if (__ldg(&pages[mid].g0) <= g) lo = mid;
    else hi = mid;
  }
  return lo;
}

// `w` bits (1 .. 64) at bit `bit` of the staged streams, LSB first: a 64-bit funnel shift of the two aligned words that
// hold them (the second is read only when the value reaches into it, so reads stay within a stream's last byte + 7)
__device__ __forceinline__ unsigned long long unpack(const unsigned long long* words, uint64_t bit, uint32_t w) {
  const uint64_t q = bit >> 6;
  const uint32_t sh = uint32_t(bit & 63);
  unsigned long long v = __ldg(words + q) >> sh;
  if (sh + w > 64) v |= __ldg(words + q + 1) << (64 - sh);
  return w == 64 ? v : (v & ((1ull << w) - 1));
}

// inclusive scan of (reset, value) pairs over the warp: a reset element starts a new sum
__device__ __forceinline__ void seg_scan(unsigned long long& v, uint32_t& f, uint32_t lane) {
#pragma unroll
  for (uint32_t o = 1; o < 32; o <<= 1) {
    const unsigned long long pv = __shfl_up_sync(FULL, v, o);
    const uint32_t pf = __shfl_up_sync(FULL, f, o);
    if (lane >= o) {
      if (!f) v += pv;
      f |= pf;
    }
  }
}

__global__ void __launch_bounds__(kThreads) k_dbp_local(const unsigned long long* __restrict__ words, const DbpPage* __restrict__ pages,
                                                         uint32_t n_pages, const DbpMini* __restrict__ mbs, uint32_t n_groups, Scratch s) {
  __shared__ unsigned long long s_tot[kDbpGroupsPerCta];
  __shared__ uint32_t s_reset[kDbpGroupsPerCta];
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t g = blockIdx.x * kDbpGroupsPerCta + warp;
  unsigned long long x = 0;
  uint32_t reset = 0;
  if (g < n_groups) {
    const uint32_t p = page_of(pages, n_pages, g);
    const uint32_t g0 = __ldg(&pages[p].g0), n = __ldg(&pages[p].n);
    const uint32_t i = (g - g0) * 32 + lane;
    if (i == 0) {
      x = __ldg(&pages[p].first);
    } else if (i < n) {
      const uint32_t per_mb = __ldg(&pages[p].per_mb);
      const uint32_t k = i - 1, m = k / per_mb, r = k - m * per_mb;
      const DbpMini* mb = mbs + __ldg(&pages[p].mb0) + m;
      const uint32_t w = __ldg(&mb->width);
      x = __ldg(&mb->min_delta);
      if (w) x += unpack(words, (__ldg(&pages[p].src) + __ldg(&mb->off)) * 8 + uint64_t(r) * w, w);
    }
    // inclusive scan of the group (lanes past the page's end add 0)
#pragma unroll
    for (uint32_t o = 1; o < 32; o <<= 1) {
      const unsigned long long y = __shfl_up_sync(FULL, x, o);
      if (lane >= o) x += y;
    }
    if (i < n) pages[p].dst[i] = x;
    reset = g == g0;
    if (lane == 0) s.grp_page[g] = p;
  }
  if (lane == 31) {
    s_tot[warp] = x;
    s_reset[warp] = reset;
  }
  __syncthreads();
  if (warp == 0) {
    const unsigned long long own = s_tot[lane];
    unsigned long long v = own;
    uint32_t f = s_reset[lane];
    seg_scan(v, f, lane);
    const uint32_t gg = blockIdx.x * kDbpGroupsPerCta + lane;
    if (gg < n_groups) s.grp_carry[gg] = v - own;  // (0 at a page start: the reset element's sum is its own)
    const unsigned any = __ballot_sync(FULL, s_reset[lane] != 0);
    if (lane == 31) {
      s.cta_sum[blockIdx.x] = v;
      s.cta_reset[blockIdx.x] = any != 0;
    }
  }
}

__global__ void __launch_bounds__(1024) k_dbp_carry(uint32_t n_ctas, Scratch s) {
  __shared__ unsigned long long s_v[32], s_in[32];
  __shared__ uint32_t s_f[32];
  __shared__ unsigned long long s_run;
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) s_run = 0;
  for (uint32_t base = 0; base < n_ctas; base += 1024) {
    const uint32_t c = base + threadIdx.x;
    const unsigned long long own = c < n_ctas ? s.cta_sum[c] : 0ull;
    const uint32_t own_f = c < n_ctas ? s.cta_reset[c] : 0u;
    unsigned long long v = own;
    uint32_t f = own_f;
    seg_scan(v, f, lane);
    if (lane == 31) {
      s_v[warp] = v;
      s_f[warp] = f;
    }
    __syncthreads();
    if (warp == 0) {
      unsigned long long wv = s_v[lane];
      uint32_t wf = s_f[lane];
      seg_scan(wv, wf, lane);
      // what enters warp `lane`: the tile's warps before it on top of the carry of the tiles before
      unsigned long long ev = __shfl_up_sync(FULL, wv, 1);
      uint32_t ef = __shfl_up_sync(FULL, wf, 1);
      if (lane == 0) {
        ev = 0;
        ef = 0;
      }
      const unsigned long long run = s_run;
      s_in[lane] = ef ? ev : run + ev;
      __syncwarp();
      if (lane == 31) s_run = wf ? wv : run + wv;
    }
    __syncthreads();
    // exclusive: the inclusive sum of the CTA before, within the warp, on top of what enters the warp
    unsigned long long ev = __shfl_up_sync(FULL, v, 1);
    uint32_t ef = __shfl_up_sync(FULL, f, 1);
    if (lane == 0) {
      ev = 0;
      ef = 0;
    }
    if (c < n_ctas) s.cta_sum[c] = ef ? ev : s_in[warp] + ev;
    __syncthreads();
  }
}

__global__ void __launch_bounds__(kThreads) k_dbp_add(const DbpPage* __restrict__ pages, uint32_t n_groups, Scratch s) {
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t g = blockIdx.x * kDbpGroupsPerCta + warp;
  if (g >= n_groups) return;
  const uint32_t p = s.grp_page[g];
  const uint32_t g0 = __ldg(&pages[p].g0), n = __ldg(&pages[p].n);
  unsigned long long carry = s.grp_carry[g];
  if (g0 < blockIdx.x * kDbpGroupsPerCta) carry += s.cta_sum[blockIdx.x];  // its page started in an earlier CTA
  const uint32_t i = (g - g0) * 32 + lane;
  if (carry != 0 && i < n) pages[p].dst[i] += carry;
}

}  // namespace

size_t dbp_scratch_bytes(uint32_t n_groups) {
  const size_t n_ctas = (size_t(n_groups) + kDbpGroupsPerCta - 1) / kDbpGroupsPerCta;
  return al16(size_t(n_groups) * 8) + al16(n_ctas * 8) + al16(size_t(n_groups) * 4) + al16(n_ctas * 4);
}

cudaError_t launch_dbp_decode(const uint8_t* stage, const DbpPage* d_pages, uint32_t n_pages, const DbpMini* d_mbs, uint32_t n_groups,
                              void* scratch, cudaStream_t st) {
  if (n_groups == 0) return cudaSuccess;
  const uint32_t n_ctas = (n_groups + kDbpGroupsPerCta - 1) / kDbpGroupsPerCta;
  const Scratch s = scratch_of(scratch, n_groups);
  k_dbp_local<<<n_ctas, kThreads, 0, st>>>(reinterpret_cast<const unsigned long long*>(stage), d_pages, n_pages, d_mbs, n_groups, s);
  k_dbp_carry<<<1, 1024, 0, st>>>(n_ctas, s);
  k_dbp_add<<<n_ctas, kThreads, 0, st>>>(d_pages, n_groups, s);
  return cudaGetLastError();
}

}  // namespace fgpu
