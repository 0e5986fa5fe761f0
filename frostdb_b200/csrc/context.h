// Engine state shared by engine.cpp and residency.cpp: the context with its stream, page-locked arena and pool, the
// error slot of the C ABI, and stream-ordered device buffers.
#pragma once
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/frostgpu.h"
#include "device_types.h"
#include "kernels.h"
#include "part_store.h"

namespace fgpu {

inline thread_local std::string g_err;  // fgpu_last_error

inline int32_t fail(int32_t code, const std::string& msg) {
  g_err = msg;
  return code;
}

#define CUDA_TRY(expr)                                                                         \
  do {                                                                                         \
    cudaError_t _e = (expr);                                                                   \
    if (_e != cudaSuccess) {                                                                   \
      cudaGetLastError();                                                                      \
      return fail(_e == cudaErrorMemoryAllocation ? FGPU_ERR_OOM : FGPU_ERR_CUDA,              \
                  std::string(#expr) + ": " + cudaGetErrorString(_e));                         \
    }                                                                                          \
  } while (0)

// Stream-ordered device allocation (cudaMallocAsync on the engine stream, pool kept warm): a query's
// scratch and a streamed part's columns cost microseconds to allocate instead of a cudaMalloc each.
struct DevBuf {
  void* p = nullptr;
  size_t n = 0;
  cudaStream_t st = nullptr;
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  ~DevBuf() { reset(); }
  void reset() {
    if (p) cudaFreeAsync(p, st);
    p = nullptr;
    n = 0;
  }
  cudaError_t alloc(size_t bytes, cudaStream_t stream) {
    reset();
    st = stream;
    if (bytes == 0) bytes = 16;
    cudaError_t e = cudaMallocAsync(&p, bytes, stream);
    if (e == cudaSuccess) n = bytes;
    else p = nullptr;
    return e;
  }
};

inline int bit_width_u32(uint64_t max_value) {
  int w = 0;
  while (w < 64 && (max_value >> w) != 0) w++;
  return w;
}

// Page-locked host blocks, recycled: result images of cached plans and the columns of large results (which the
// Arrow consumer holds until it releases the array, possibly after the context is gone: the pool is shared-owned).
// Freeing page-locked memory synchronises the device, so blocks are only released when the pool itself dies.
struct PinnedPool {
  std::mutex mu;
  std::multimap<size_t, uint8_t*> free_blocks;
  size_t free_bytes = 0;
  ~PinnedPool() {
    for (auto& kv : free_blocks) cudaFreeHost(kv.second);
  }
  uint8_t* take(size_t bytes, size_t* cap) {
    size_t want = 4096;
    while (want < bytes) want <<= 1;
    if (bytes > (size_t(1) << 24)) want = (bytes + (size_t(1) << 22) - 1) & ~((size_t(1) << 22) - 1);  // large blocks: 4 MiB granules
    {
      std::lock_guard<std::mutex> lk(mu);
      auto it = free_blocks.lower_bound(want);
      if (it != free_blocks.end() && it->first <= want * 2) {
        uint8_t* p = it->second;
        *cap = it->first;
        free_bytes -= it->first;
        free_blocks.erase(it);
        return p;
      }
    }
    uint8_t* p = nullptr;
    if (cudaHostAlloc(reinterpret_cast<void**>(&p), want, cudaHostAllocDefault) != cudaSuccess) {
      cudaGetLastError();
      return nullptr;
    }
    *cap = want;
    return p;
  }
  void give(uint8_t* p, size_t cap) {
    std::lock_guard<std::mutex> lk(mu);
    free_blocks.emplace(cap, p);
    free_bytes += cap;
  }
};

// One block of a PinnedPool, owned: it goes back to its pool when its owner is destroyed, so no return path can
// lose it.  A block that becomes Arrow buffers moves into keep(), which a column holds as its ext_keep.
class PinnedBlock {
 public:
  PinnedBlock() = default;
  PinnedBlock(const std::shared_ptr<PinnedPool>& pool, size_t bytes) : pool_(pool) { p_ = pool->take(bytes, &cap_); }  // empty when out of memory
  PinnedBlock(PinnedBlock&& o) noexcept : pool_(std::move(o.pool_)), p_(o.p_), cap_(o.cap_) { o.p_ = nullptr; }
  PinnedBlock& operator=(PinnedBlock&& o) noexcept {  // returns the block it held, takes o's
    if (this != &o) {
      reset();
      pool_ = std::move(o.pool_);
      p_ = o.p_;
      cap_ = o.cap_;
      o.p_ = nullptr;
    }
    return *this;
  }
  ~PinnedBlock() { reset(); }
  uint8_t* get() const { return p_; }
  explicit operator bool() const { return p_ != nullptr; }
  // The block, shared: it returns to the pool when the last holder lets go (the consumer released every array).
  std::shared_ptr<void> keep() && { return std::make_shared<PinnedBlock>(std::move(*this)); }

 private:
  void reset() {
    if (p_) pool_->give(p_, cap_);
    p_ = nullptr;
  }
  std::shared_ptr<PinnedPool> pool_;
  uint8_t* p_ = nullptr;
  size_t cap_ = 0;
};

constexpr size_t kCommDataOff = 4096;  // flags live in front of the slots

// Mailbox communicator of one rank (see comm.cu).
struct Comm {
  int rank = -1, n = 0;
  uint64_t slot_bytes = 0, total = 0, seq = 0;
  uint8_t* mailbox = nullptr;  // [flags: 2 sets x kMaxRanks x {seq, bytes}] ... [2 sets x n slots]
  bool open = false;
  uint8_t* peer[kMaxRanks] = {nullptr};
  bool peer_ipc[kMaxRanks] = {false};
  size_t flag_off(uint64_t set, int r) const { return (size_t(set) * kMaxRanks + size_t(r)) * 16; }
  size_t data_off(uint64_t set, int r) const { return kCommDataOff + (size_t(set) * size_t(n) + size_t(r)) * slot_bytes; }
};

}  // namespace fgpu

struct fgpu_ctx {
  fgpu::Comm comm;
  int device = 0;
  int sm_count = 132;
  int tile_rows = fgpu::kTileRows;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
  std::mutex mu;
  std::map<std::string, fgpu::Table> tables;
  std::vector<fgpu::ColumnImage*> pending_uploads;  // staging to release after the next stream sync
  uint64_t epoch_counter = 0;                 // source of Table::epoch stamps
  std::map<std::string, std::shared_ptr<struct QueryPlan>> plans;  // by plan signature (bounded, see fgpu_query_prepare)
  // page-locked arena for column metadata on its way to the device: a pageable source would make every
  // cudaMemcpyAsync wait for the transfers queued before it.  Reset by release_staging() after a sync.
  uint8_t* arena = nullptr;
  size_t arena_cap = 0, arena_used = 0;
  void* arena_take(size_t n) {
    if (!arena) {
      size_t want = size_t(64) << 20;
      if (cudaHostAlloc(reinterpret_cast<void**>(&arena), want, cudaHostAllocDefault) != cudaSuccess) {
        cudaGetLastError();
        arena = nullptr;
        return nullptr;
      }
      arena_cap = want;
    }
    size_t off = (arena_used + 63) & ~size_t(63);
    if (off + n > arena_cap) return nullptr;  // caller falls back to the pageable source
    arena_used = off + n;
    return arena + off;
  }
  std::shared_ptr<fgpu::PinnedPool> pinned = std::make_shared<fgpu::PinnedPool>();  // blocks are taken as PinnedBlock
  // page-locked scratch for the per-query descriptor upload and the counters read-back (guarded by mu)
  uint8_t* scratch = nullptr;
  size_t scratch_bytes = 0;
  cudaError_t ensure_scratch(size_t bytes) {
    if (bytes <= scratch_bytes) return cudaSuccess;
    if (scratch) cudaFreeHost(scratch);
    scratch = nullptr;
    scratch_bytes = 0;
    size_t want = std::max<size_t>(bytes * 2, 1 << 20);
    cudaError_t e = cudaHostAlloc(reinterpret_cast<void**>(&scratch), want, cudaHostAllocDefault);
    if (e == cudaSuccess) scratch_bytes = want;
    return e;
  }
};
