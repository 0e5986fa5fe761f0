// Non-dictionary string pages of Parquet parts (PLAIN, DELTA_LENGTH_BYTE_ARRAY, DELTA_BYTE_ARRAY) interned at upload
// (sm_90a).  The host's page walk has validated every value and left its address; one batch covers every chunk with
// such values of a call that makes columns resident:
//   k_str_unfront  one warp per run of up to kFrontSeg values of a DELTA_BYTE_ARRAY page, 32 values at a time, one
//                  lane per value: byte j of value i is suffix byte j - pre[k] of k = max{k <= i : pre[k] <= j} (one
//                  ballot over the window); when no k of the window qualifies it is byte j of the value before the
//                  window, which the warp rebuilt in its previous step, or, for a run's first window, which a backward
//                  ballot search finds (windows of 32 least prefix lengths, then one window of prefix lengths).
//   k_str_hash     one thread per value: XXH64 of its bytes, then linear probing in its chunk's open-addressing table.
//                  A slot is claimed by CAS with (hash >> 32, value index); a value whose hash matches compares length
//                  and bytes with the slot's representative and probes on when they differ, so two strings share a
//                  slot only when their bytes are equal.  atomicMin keeps the slot's first occurrence.
//   k_str_compact  one thread per slot: every used slot gets a dense rank per chunk and its first occurrence goes to
//                  the host (page-locked memory, 4 bytes per distinct value).  The host sorts them, interns the new
//                  strings in that order and uploads the chunk-local index per rank.
//   k_str_gather   one thread per slot of the chunks with DELTA_BYTE_ARRAY values, one warp per value copied: the bytes
//                  of every distinct rebuilt value's first occurrence go to page-locked memory, where the host interns
//                  them from (PLAIN and DELTA_LENGTH_BYTE_ARRAY values it interns from the file bytes it walked).
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

// value v of a chunk: its bytes and length, behind a length prefix (PLAIN pages only) or addressed by start and length
__device__ __forceinline__ const uint8_t* value_at(const StrChunk& c, uint32_t v, uint32_t* len) {
  const uint8_t* p = c.bytes + c.off[v];
  if (c.len) {
    *len = c.len[v];
    return p;
  }
  *len = rd32(p);
  return p + 4;
}

// byte b of value x of a DELTA_BYTE_ARRAY page (x relative to the page), found by the whole warp (x and b warp-uniform):
// the last value k <= x whose prefix is at most b holds it in its suffix.  The page's first prefix is 0, so k exists.
__device__ uint8_t front_byte(const StrChunk& c, const StrFrontJob& j, uint32_t x, uint32_t b, uint32_t lane) {
  const uint32_t* pre = c.pre + j.d0;
  uint32_t w = x / 32;
  unsigned m = __ballot_sync(FULL, w * 32 + lane <= x && pre[w * 32 + lane] <= b);
  if (m == 0) {  // the nearest earlier window holding such a prefix, 32 windows per step
    unsigned mw;
    for (;;) {
      const int ww = int(w) - 1 - int(lane);
      mw = __ballot_sync(FULL, ww >= 0 && c.wmin[j.w0 + uint32_t(ww)] <= b);
      if (mw) break;
      w -= 32;
    }
    w = w - 1 - uint32_t(__ffs(mw) - 1);
    m = __ballot_sync(FULL, pre[w * 32 + lane] <= b);  // (a window before x's window is whole)
  }
  const uint32_t k = w * 32 + 31 - uint32_t(__clz(m));
  return c.bytes[c.suf[j.d0 + k] + b - pre[k]];
}

__global__ void __launch_bounds__(kThreads) k_str_unfront(const StrChunk* __restrict__ chunks, const StrFrontJob* __restrict__ jobs,
                                                          uint32_t n_jobs) {
  const uint32_t wid = (blockIdx.x * blockDim.x + threadIdx.x) / 32u;
  const uint32_t lane = threadIdx.x & 31u;
  if (wid >= n_jobs) return;  // (warp-uniform)
  const StrFrontJob j = jobs[wid];
  const StrChunk& c = chunks[j.chunk];
  uint8_t* const bytes = c.bytes;
  const unsigned upto = lane == 31 ? FULL : (2u << lane) - 1u;  // lanes <= this one
  for (uint32_t base = j.seg; base < j.seg + j.n; base += 32) {
    const uint32_t x = base + lane;
    uint32_t p = FULL, len = 0, suf = 0, out = 0;
    if (x < j.seg + j.n) {
      p = c.pre[j.d0 + x];
      suf = c.suf[j.d0 + x];
      len = c.len[j.v0 + x];
      out = c.off[j.v0 + x];
    }
    const uint32_t max_len = __reduce_max_sync(FULL, len);
    for (uint32_t b = 0; b < max_len; b++) {
      const unsigned m = __ballot_sync(FULL, p <= b) & upto;
      const int k = m ? 31 - __clz(m) : 0;
      const uint32_t ks = __shfl_sync(FULL, suf, k), kp = __shfl_sync(FULL, p, k);
      const bool before = b < len && m == 0;  // byte b of the value before the window
      uint8_t v = 0;
      if (__any_sync(FULL, before)) {
        if (base > j.seg) v = bytes[c.off[j.v0 + base - 1] + b];  // rebuilt by this warp's previous step
        else v = front_byte(c, j, base - 1, b, lane);
      }
      if (b < len) bytes[out + b] = before ? v : bytes[ks + b - kp];
    }
    __syncwarp();  // the window's values are visible to the next step
  }
}

__global__ void __launch_bounds__(kThreads) k_str_hash(const StrChunk* __restrict__ chunks, uint32_t n_chunks, uint32_t total) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= total) return;
  const StrChunk& c = chunks[chunk_of(chunks, n_chunks, t, false)];
  const uint32_t v = t - c.v0;
  uint32_t len;
  const uint8_t* s = value_at(c, v, &len);
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
      uint32_t rlen;
      const uint8_t* r = value_at(c, uint32_t(k), &rlen);
      bool eq = rlen == len;
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

__global__ void __launch_bounds__(kThreads) k_str_gather(const StrChunk* __restrict__ chunks, uint32_t n_chunks, uint32_t total) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t lane = threadIdx.x & 31u;
  const uint8_t* src = nullptr;
  uint8_t* dst = nullptr;
  uint32_t len = 0;
  if (t < total) {
    const StrChunk& c = chunks[chunk_of(chunks, n_chunks, t, true)];
    const uint32_t s = t - c.s0;
    if (c.out_rebuilt && c.keys[s] != kEmpty) {
      const uint32_t f = c.out_first[c.first[s]];  // (first is the slot's rank now)
      const uint32_t off = c.off[f];
      if (off >= c.rb0) {
        src = c.bytes + off;
        dst = c.out_rebuilt + (off - c.rb0);
        len = c.len[f];
      }
    }
  }
  for (unsigned todo = __ballot_sync(FULL, len > 0); todo; todo &= todo - 1) {  // the warp copies one value at a time
    const int l = __ffs(todo) - 1;
    const uint8_t* s = reinterpret_cast<const uint8_t*>(__shfl_sync(FULL, reinterpret_cast<unsigned long long>(src), l));
    uint8_t* d = reinterpret_cast<uint8_t*>(__shfl_sync(FULL, reinterpret_cast<unsigned long long>(dst), l));
    const uint32_t n = __shfl_sync(FULL, len, l);
    for (uint32_t i = lane; i < n; i += 32) d[i] = s[i];
  }
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

cudaError_t launch_str_unfront(const StrChunk* d_chunks, const StrFrontJob* d_jobs, uint32_t n_jobs, cudaStream_t st) {
  if (n_jobs == 0) return cudaSuccess;
  k_str_unfront<<<blocks_for(n_jobs * 32u), kThreads, 0, st>>>(d_chunks, d_jobs, n_jobs);
  return cudaGetLastError();
}

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

cudaError_t launch_str_gather(const StrChunk* d_chunks, uint32_t n_chunks, uint32_t total_slots, cudaStream_t st) {
  if (n_chunks == 0 || total_slots == 0) return cudaSuccess;
  k_str_gather<<<blocks_for(total_slots), kThreads, 0, st>>>(d_chunks, n_chunks, total_slots);
  return cudaGetLastError();
}

cudaError_t launch_str_codes(const StrCodeJob* d_jobs, uint32_t n_jobs, uint32_t total_groups, cudaStream_t st) {
  if (n_jobs == 0 || total_groups == 0) return cudaSuccess;
  k_str_codes<<<blocks_for(total_groups), kThreads, 0, st>>>(d_jobs, n_jobs, total_groups);
  return cudaGetLastError();
}

}  // namespace fgpu
