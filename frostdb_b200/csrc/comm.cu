// Partial-table exchange between the GPUs of one node, inside the library (sm_90a): the step the reference runs
// as per-goroutine partial HashAggregate -> Synchronizer -> final HashAggregate (physicalplan.go:438-471,
// synchronize.go:16-53), with one process (or one context) per GPU.
//
// Every rank owns a MAILBOX in its HBM: two sets (by sequence parity) of one slot per rank, plus one flag per set
// and rank.  Peers map each other's mailboxes (CUDA IPC between processes, plain peer access inside one process).
// One collective Execute enqueues, on the rank's one stream and behind its scan:
//   k_comm_push    the rank's partial aggregate table goes into slot [my rank] of EVERY rank's mailbox with
//                  16-byte stores over NVLink (no host, no NCCL launch on the critical path); the last CTA to finish
//                  raises flag[my rank] = sequence number in every mailbox (system fence + st.release.sys: the
//                  pushed bytes are visible before the flag);
//   k_finalize_dense (kernels.cu, cached dense plans) waits in every CTA with ld.acquire.sys until every rank's flag of
//                  this set carries the sequence number (bounded by a timeout, reported through the query's
//                  counters), then compacts the FOLD of the n mailbox slots into the result columns: wait, merge and
//                  finalize are one launch;
//   k_comm_wait + k_merge_dense  the same in two launches for the plans without an execution cache (the final table is
//                  written back; hash tables go through k_merge per rank, kernels.cu).  Dense tables have the same
//                  shape on every rank, which k_comm_wait checks; a hash table is sized from its rank's own rows, so
//                  the host reads the pushed byte counts behind the wait and sizes the merge table from them.
// Double buffering by sequence parity is enough: a rank can only push sequence k + 2 after it merged k + 1, which
// needed every peer's push k + 1, which every peer enqueued behind its own merge of k.
#include <cuda_runtime.h>

#include "agg_ops.cuh"
#include "device_types.h"
#include "kernels.h"

namespace fgpu {
namespace {

__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_sys(unsigned long long* p, unsigned long long v) {
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long global_timer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}

__global__ void __launch_bounds__(256) k_comm_push(CommPush p) {
  const uint4* src = reinterpret_cast<const uint4*>(p.src);
  const size_t n16 = p.bytes / 16, stride = size_t(gridDim.x) * blockDim.x;
  for (size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n16; i += stride) {
    const uint4 v = src[i];
#pragma unroll 4
    for (int r = 0; r < p.n; r++) reinterpret_cast<uint4*>(p.dst[r])[i] = v;
  }
  // the last CTA to finish raises the flags: one release-ordered system-scope store per peer, behind a system fence
  // of every CTA's copies (no second launch between the copies and the signal)
  __shared__ bool last;
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence_system();  // cumulative over the CTA's stores (ordered before it by the barrier): one fence per CTA, not per thread
    last = atomicAdd(p.done, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (last) {
    __threadfence_system();
    const int r = threadIdx.x;
    if (r < p.n) {
      p.flag[r][1] = p.bytes;  // what was pushed (checked by the receiver against its own table shape)
      __threadfence_system();
      st_release_sys(p.flag[r], p.seq);
    }
    if (threadIdx.x == 0) *p.done = 0;
  }
}

__global__ void k_comm_wait(CommWait w) {
  const int r = threadIdx.x;
  bool timeout = false, mismatch = false;
  if (r < w.n) {
    const unsigned long long t0 = global_timer_ns();
    while (ld_acquire_sys(w.flags + 2 * r) < w.seq) {
      __nanosleep(200);
      if (global_timer_ns() - t0 > w.timeout_ns) { timeout = true; break; }
    }
    if (!timeout && w.bytes != 0 && w.flags[2 * r + 1] != w.bytes) mismatch = true;
  }
  if (timeout) atomicExch(w.counters + 3, 1ull);
  else if (mismatch) atomicExch(w.counters + 3, 2ull);
}

// final table = fold over the ranks' partial tables (layout of table_layout(): [rows][stored aggregates...])
__global__ void __launch_bounds__(256) k_merge_dense(QueryDesc q, CommMerge m) {
  if (q.counters[3] != 0) return;  // the exchange failed: leave the local table alone
  const size_t S = q.table_slots, stride = size_t(gridDim.x) * blockDim.x;
  for (size_t s = size_t(blockIdx.x) * blockDim.x + threadIdx.x; s < S; s += stride) {
    unsigned long long rows = 0;
    for (int r = 0; r < m.n; r++) rows += reinterpret_cast<const unsigned long long*>(m.src[r])[s];
    q.t_rows[s] = rows;
    int pos = 0;
    for (int a = 0; a < q.n_aggs; a++) {
      const AggDesc ad = q.aggs[a];
      if (ad.func == 4) continue;
      long long v = agg_identity(ad.func, ad.is_float);
      for (int r = 0; r < m.n; r++) {
        if (reinterpret_cast<const unsigned long long*>(m.src[r])[s] == 0) continue;  // an empty group holds the identity, not a value
        v = agg_combine(ad.func, ad.is_float, v, reinterpret_cast<const long long*>(m.src[r] + S * 8 * size_t(1 + pos))[s]);
      }
      q.t_agg[a][s] = v;
      pos++;
    }
  }
}

}  // namespace

cudaError_t launch_comm_push(const CommPush& p, int sm_count, cudaStream_t st) {
  size_t blocks = (p.bytes / 16 + 255) / 256;
  if (blocks > size_t(sm_count) * 2) blocks = size_t(sm_count) * 2;
  if (blocks < 1) blocks = 1;
  k_comm_push<<<unsigned(blocks), 256, 0, st>>>(p);
  return cudaGetLastError();
}

cudaError_t launch_comm_wait(const CommWait& w, cudaStream_t st) {
  k_comm_wait<<<1, 32, 0, st>>>(w);
  return cudaGetLastError();
}

cudaError_t launch_merge_dense(const QueryDesc& q, const CommMerge& m, cudaStream_t st) {
  size_t blocks = (size_t(q.table_slots) + 255) / 256;
  if (blocks > 132 * 4) blocks = 132 * 4;  // 4 CTAs per SM of an H100 SXM (132 SMs), grid-stride beyond
  if (blocks < 1) blocks = 1;
  k_merge_dense<<<unsigned(blocks), 256, 0, st>>>(q, m);
  return cudaGetLastError();
}

}  // namespace fgpu
