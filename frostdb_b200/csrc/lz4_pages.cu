// LZ4_RAW-compressed PLAIN INT64 / DOUBLE pages of Parquet parts inflated at upload into the dense value array (sm_90a).
// The host's page walk has validated every block against its page's inflated size (parse_lz4_raw); the blocks sit in the
// upload's staging buffer and every page's values are a hole in the column image.  The sequence chain of a block is
// serial by format (a sequence starts where the one before it ends), so the unit of work is one page per warp:
//   - every lane decodes a sequence's token, length extensions and offset from the same bytes (broadcast loads);
//   - the warp copies the literals lane-parallel, in 16-byte pieces when source and hole share their alignment;
//   - the warp copies the match lane-parallel: a match that does not overlap its source like the literals, an overlapping
//     one (offset < length) as the repetition of the `offset` bytes before it, lane i writing byte pos + i + 32 k from
//     byte pos - offset + (i + 32 k) mod offset, so that no lane reads a byte the same match writes.
// The kernel trusts the host's validation, yet bounds every write to the page's hole and every read to its staged block.
#include <cuda_runtime.h>

#include "device_types.h"
#include "kernels.h"

namespace fgpu {
namespace {

// n bytes from src to dst (not overlapping), lane-parallel
__device__ __forceinline__ void warp_copy(unsigned char* dst, const unsigned char* src, uint32_t n, uint32_t lane) {
  uint32_t i0 = 0;
  if (((reinterpret_cast<uintptr_t>(dst) ^ reinterpret_cast<uintptr_t>(src)) & 15) == 0 && n >= 64) {
    const uint32_t head = (16u - uint32_t(reinterpret_cast<uintptr_t>(dst) & 15)) & 15u;
    if (lane < head) dst[lane] = src[lane];
    const uint32_t body = (n - head) / 16;
    uint4* d = reinterpret_cast<uint4*>(dst + head);
    const uint4* s = reinterpret_cast<const uint4*>(src + head);
    for (uint32_t i = lane; i < body; i += 32) d[i] = s[i];
    i0 = head + body * 16;
  }
  for (uint32_t i = i0 + lane; i < n; i += 32) dst[i] = src[i];
}

__global__ void __launch_bounds__(32 * kLz4WarpsPerCta) k_lz4_pages(const unsigned char* __restrict__ stage, const Lz4Job* __restrict__ jobs,
                                                                    uint32_t n_jobs) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t j = blockIdx.x * kLz4WarpsPerCta + (threadIdx.x >> 5);
  if (j >= n_jobs) return;
  const unsigned char* src = stage + jobs[j].src;
  unsigned char* dst = jobs[j].dst;
  const uint32_t len = jobs[j].len, cap = jobs[j].out_len;
  uint32_t ip = 0, op = 0;
  while (ip < len && op < cap) {
    const uint32_t token = src[ip++];
    uint32_t lit = token >> 4;
    if (lit == 15)
      for (uint32_t b = 255; b == 255 && ip < len;) lit += (b = src[ip++]);
    lit = min(lit, len - ip);
    const uint32_t nl = min(lit, cap - op);
    warp_copy(dst + op, src + ip, nl, lane);
    ip += lit;
    op += nl;
    if (ip + 2 > len || op >= cap) break;  // the last sequence has no match
    const uint32_t offset = uint32_t(src[ip]) | (uint32_t(src[ip + 1]) << 8);
    ip += 2;
    uint32_t ml = token & 15u;
    if (ml == 15)
      for (uint32_t b = 255; b == 255 && ip < len;) ml += (b = src[ip++]);
    ml = min(ml + 4, cap - op);
    if (offset == 0 || offset > op) break;
    __syncwarp();  // the bytes before `op` that other lanes wrote are visible
    if (offset >= ml) {
      warp_copy(dst + op, dst + op - offset, ml, lane);
    } else {
      const unsigned char* from = dst + op - offset;
      const uint32_t step = 32u % offset;
      uint32_t r = lane % offset;
      for (uint32_t k = lane; k < ml; k += 32) {
        dst[op + k] = from[r];
        r += step;
        if (r >= offset) r -= offset;
      }
    }
    op += ml;
  }
}

}  // namespace

cudaError_t launch_lz4_pages(const uint8_t* stage, const Lz4Job* d_jobs, uint32_t n_jobs, cudaStream_t st) {
  if (n_jobs == 0) return cudaSuccess;
  const uint32_t ctas = (n_jobs + kLz4WarpsPerCta - 1) / kLz4WarpsPerCta;
  k_lz4_pages<<<ctas, 32 * kLz4WarpsPerCta, 0, st>>>(stage, d_jobs, n_jobs);
  return cudaGetLastError();
}

}  // namespace fgpu
