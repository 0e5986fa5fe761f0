// PLAIN string pages of Parquet parts interned at upload (sm_90a).  The host's page walk has validated every length
// prefix and left one offset per value; one batch covers every chunk with PLAIN string values of a call that makes
// columns resident:
//   k_str_hash     one thread per value: XXH64 of its bytes, then linear probing in its chunk's open-addressing table.
//                  A slot is claimed by CAS with (hash >> 32, value index); a value whose hash matches compares length
//                  and bytes with the slot's representative and probes on when they differ, so two strings share a
//                  slot only when their bytes are equal.  atomicMin keeps the slot's first occurrence.
//   k_str_compact  one thread per slot: every used slot gets a dense rank per chunk and its first occurrence goes to
//                  the host (page-locked memory, 4 bytes per distinct value).  The host sorts them, interns the new
//                  strings in that order (from the file bytes it walked) and uploads the chunk-local index per rank.
//   k_str_codes    one thread per 8 values of a page (one whole byte group at any width): the values' chunk-local
//                  indices, packed LSB first at the chunk's width into the hole the page owns in the resident image.
#include <cuda_runtime.h>

#include "device_types.h"
#include "kernels.h"

namespace fgpu {
namespace {

constexpr unsigned FULL = 0xffffffffu;
constexpr unsigned long long kEmpty = ~0ull;
constexpr int kThreads = 256;

// values sit at any byte alignment
__device__ __forceinline__ uint64_t rd64(const uint8_t* p) {
  uint64_t v = 0;
#pragma unroll
  for (int i = 0; i < 8; i++) v |= uint64_t(p[i]) << (8 * i);
  return v;
}
__device__ __forceinline__ uint32_t rd32(const uint8_t* p) {
  return uint32_t(p[0]) | (uint32_t(p[1]) << 8) | (uint32_t(p[2]) << 16) | (uint32_t(p[3]) << 24);
}

constexpr uint64_t kP1 = 11400714785074694791ull, kP2 = 14029467366897019727ull, kP3 = 1609587929392839161ull,
                   kP4 = 9650029242287828579ull, kP5 = 2870177450012600261ull;
__device__ __forceinline__ uint64_t rotl64(uint64_t x, int r) { return (x << r) | (x >> (64 - r)); }
__device__ __forceinline__ uint64_t xx_round(uint64_t acc, uint64_t in) { return rotl64(acc + in * kP2, 31) * kP1; }
__device__ __forceinline__ uint64_t xx_merge(uint64_t acc, uint64_t v) { return (acc ^ xx_round(0, v)) * kP1 + kP4; }

// XXH64, seed 0 (the host's xxhash64 in parquet_meta.cpp)
__device__ uint64_t xxh64(const uint8_t* p, uint32_t len) {
  const uint8_t* const end = p + len;
  uint64_t h;
  if (len >= 32) {
    uint64_t v1 = kP1 + kP2, v2 = kP2, v3 = 0, v4 = 0 - kP1;
    do {
      v1 = xx_round(v1, rd64(p));
      v2 = xx_round(v2, rd64(p + 8));
      v3 = xx_round(v3, rd64(p + 16));
      v4 = xx_round(v4, rd64(p + 24));
      p += 32;
    } while (p + 32 <= end);
    h = rotl64(v1, 1) + rotl64(v2, 7) + rotl64(v3, 12) + rotl64(v4, 18);
    h = xx_merge(h, v1);
    h = xx_merge(h, v2);
    h = xx_merge(h, v3);
    h = xx_merge(h, v4);
  } else {
    h = kP5;
  }
  h += uint64_t(len);
  while (p + 8 <= end) {
    h ^= xx_round(0, rd64(p));
    h = rotl64(h, 27) * kP1 + kP4;
    p += 8;
  }
  if (p + 4 <= end) {
    h ^= uint64_t(rd32(p)) * kP1;
    h = rotl64(h, 23) * kP2 + kP3;
    p += 4;
  }
  while (p < end) {
    h ^= uint64_t(*p) * kP5;
    h = rotl64(h, 11) * kP1;
    p++;
  }
  h ^= h >> 33;
  h *= kP2;
  h ^= h >> 29;
  h *= kP3;
  h ^= h >> 32;
  return h;
}

// the chunk that holds batch ordinal t: the last one whose base is <= t (bases ascend from 0)
__device__ __forceinline__ uint32_t chunk_of(const StrChunk* chunks, uint32_t n, uint32_t t, bool slots) {
  uint32_t lo = 0, hi = n;
  while (hi - lo > 1) {
    const uint32_t mid = (lo + hi) >> 1;
    if ((slots ? chunks[mid].s0 : chunks[mid].v0) <= t) lo = mid;
    else hi = mid;
  }
  return lo;
}

__global__ void __launch_bounds__(kThreads) k_str_hash(const StrChunk* __restrict__ chunks, uint32_t n_chunks, uint32_t total) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= total) return;
  const StrChunk& c = chunks[chunk_of(chunks, n_chunks, t, false)];
  const uint32_t v = t - c.v0;
  const uint8_t* bytes = c.bytes;
  const uint8_t* s = bytes + c.off[v];
  const uint32_t len = rd32(s);
  s += 4;
  const uint64_t h = xxh64(s, len);
  const uint32_t tag = uint32_t(h >> 32);
  const uint32_t mask = c.mask;
  unsigned long long* keys = c.keys;
  uint32_t slot = uint32_t(h) & mask;
  for (;;) {  // the table holds at least twice the chunk's values: a free slot is always ahead
    unsigned long long k = *reinterpret_cast<volatile unsigned long long*>(keys + slot);
    if (k == kEmpty) {
      k = atomicCAS(keys + slot, kEmpty, (static_cast<unsigned long long>(tag) << 32) | v);
      if (k == kEmpty) break;  // claimed: this value represents the slot
    }
    if (uint32_t(k >> 32) == tag) {
      const uint8_t* r = bytes + c.off[uint32_t(k)];
      bool eq = rd32(r) == len;
      r += 4;
      for (uint32_t i = 0; eq && i < len; i++) eq = r[i] == s[i];
      if (eq) break;
    }
    slot = (slot + 1) & mask;
  }
  atomicMin(c.first + slot, v);
  c.slot[v] = slot;
}

__global__ void __launch_bounds__(kThreads) k_str_compact(const StrChunk* __restrict__ chunks, uint32_t n_chunks, uint32_t total,
                                                          uint32_t* __restrict__ counts) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t lane = threadIdx.x & 31u;
  uint32_t ci = 0, s = 0;
  bool used = false;
  if (t < total) {
    ci = chunk_of(chunks, n_chunks, t, true);
    s = t - chunks[ci].s0;
    used = chunks[ci].keys[s] != kEmpty;
  }
  const unsigned m = __ballot_sync(FULL, used);
  if (!used) return;
  const unsigned peers = __match_any_sync(m, ci);  // one atomic per chunk and warp
  const int leader = __ffs(peers) - 1;
  uint32_t base = 0;
  if (int(lane) == leader) base = atomicAdd(counts + ci, uint32_t(__popc(peers)));
  base = __shfl_sync(peers, base, leader);
  const uint32_t pos = base + uint32_t(__popc(peers & ((1u << lane) - 1u)));
  const StrChunk& c = chunks[ci];
  c.out_first[pos] = c.first[s];
  c.first[s] = pos;
}

__global__ void __launch_bounds__(kThreads) k_str_codes(const StrCodeJob* __restrict__ jobs, uint32_t n_jobs, uint32_t total) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= total) return;
  uint32_t lo = 0, hi = n_jobs;
  while (hi - lo > 1) {
    const uint32_t mid = (lo + hi) >> 1;
    if (jobs[mid].g0 <= t) lo = mid;
    else hi = mid;
  }
  const StrCodeJob& j = jobs[lo];
  const uint32_t g = t - j.g0, v0 = g * 8u, w = j.w;
  uint8_t* dst = j.dst + size_t(g) * w;
  uint64_t acc = 0;
  uint32_t bits = 0;
#pragma unroll
  for (uint32_t k = 0; k < 8; k++) {
    const uint32_t code = v0 + k < j.n ? __ldg(j.code + __ldg(j.rank + __ldg(j.slot + v0 + k))) : 0u;
    acc |= uint64_t(code) << bits;
    bits += w;
    while (bits >= 8) {
      *dst++ = uint8_t(acc);
      acc >>= 8;
      bits -= 8;
    }
  }
}

unsigned blocks_for(uint32_t n) { return (n + kThreads - 1) / kThreads; }

}  // namespace

cudaError_t launch_str_hash(const StrChunk* d_chunks, uint32_t n_chunks, uint32_t total_values, cudaStream_t st) {
  if (n_chunks == 0 || total_values == 0) return cudaSuccess;
  k_str_hash<<<blocks_for(total_values), kThreads, 0, st>>>(d_chunks, n_chunks, total_values);
  return cudaGetLastError();
}

cudaError_t launch_str_compact(const StrChunk* d_chunks, uint32_t n_chunks, uint32_t total_slots, uint32_t* d_counts, cudaStream_t st) {
  if (n_chunks == 0 || total_slots == 0) return cudaSuccess;
  k_str_compact<<<blocks_for(total_slots), kThreads, 0, st>>>(d_chunks, n_chunks, total_slots, d_counts);
  return cudaGetLastError();
}

cudaError_t launch_str_codes(const StrCodeJob* d_jobs, uint32_t n_jobs, uint32_t total_groups, cudaStream_t st) {
  if (n_jobs == 0 || total_groups == 0) return cudaSuccess;
  k_str_codes<<<blocks_for(total_groups), kThreads, 0, st>>>(d_jobs, n_jobs, total_groups);
  return cudaGetLastError();
}

}  // namespace fgpu
