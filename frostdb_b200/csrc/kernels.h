// Launch interface of kernels.cu (host side).
#pragma once
#include <cuda_runtime.h>

#include <cstddef>
#include <cstdint>

#include "device_types.h"

namespace fgpu {

constexpr int kScanThreads = 256;
constexpr int kRowsPerThread = 4;
constexpr int kTileRows = kScanThreads * kRowsPerThread;  // 1024 rows per CTA iteration
constexpr int kVecThreads = 128;  // scan kernel: 4 independent warps per CTA
constexpr int kMaxVecRows = 1024;  // rows per warp vector (multiple of kIndexRows)
constexpr int kIndexRows = 128;  // chunk index granularity (one warp): fixed when run directories are built

// Launch configuration of a kernel on the current device, cached per (device, kernel) behind one mutex: raise its
// dynamic shared memory limit to at least `smem` bytes, and its resident CTAs per SM at (threads, smem), at least 1.
cudaError_t kernel_smem_at_least(const void* kern, size_t smem);
cudaError_t kernel_ctas_per_sm(const void* kern, int threads, size_t smem, int* per_sm);

cudaError_t launch_table_init(const QueryDesc& q, cudaStream_t st, bool zero_counters = true);
cudaError_t launch_scan(const QueryDesc* d_q, const QueryDesc& q, int sm_count, cudaStream_t st);
// sorted-run scan, CTA-cooperative with TMA-staged column tiles (runs_tma.cu): nl range leaves, nk run-length keys,
// na Sum / Min / Max aggregates
uint32_t runs_tma_tile_rows(uint32_t tile_bytes, uint32_t row_bytes, uint32_t n_rows, uint32_t max_runs);  // rows per tile of one row group
void runs_tma_plan(RunsDesc& d, int nq, uint32_t max_tile, uint32_t col_region, int force_stages, int force_warps, int force_chunk);  // ring depth, stage layout
size_t runs_tma_smem_bytes(const RunsDesc& d);
int runs_tma_ctas_per_sm(const RunsDesc& d);
cudaError_t launch_runs_tma(const RunsDesc& d, int nl, int nk, int na, int sm_count, cudaStream_t st);
// all-pass sorted row groups from the key run directories and prefix-sum images (runs_prefix.cu)
uint32_t runs_prefix_window_rows(uint32_t n_rows, uint32_t sum_runs);  // rows per window of one row group
// build step of a plan's segment table: `scratch` of prefix_build_scratch_bytes(n_slots) bytes; the table's segment
// count ends up in seg_off[n_slots]
size_t prefix_build_scratch_bytes(uint32_t n_slots);
cudaError_t launch_prefix_build(PrefixBuildDesc d, uint32_t n_slots, uint32_t* seg_off, void* scratch, int sm_count, cudaStream_t st);
cudaError_t launch_runs_prefix(const PrefixDesc& d, int sm_count, cudaStream_t st);
// filter-only plans over PLAIN columns (take_rows.cu): count per span, scan, ordered write
cudaError_t launch_take(const TakeDesc& d, int sm_count, cudaStream_t st);
int take_resident_warps(int sm_count);
// tile aggregate (tile_agg.cu): TMA-staged column tiles, CTA-private shared-memory table
cudaError_t launch_tile_agg(const TileAggDesc& d, int sm_count, cudaStream_t st);
size_t tile_agg_smem_bytes(const TileAggDesc& d);
// dictionary column chunks -> flat code arrays (kernels.cu)
cudaError_t launch_flatten(const FlatJob* d_jobs, uint32_t n_jobs, uint32_t total_blocks, int sm_count, cudaStream_t st);
// PLAIN int64 column chunks -> frame-of-reference and prefix-sum images (kernels.cu): min / max per job and the sum of
// every block, then the narrowing / prefix pass
cudaError_t launch_chunk_minmax(const NarrowJob* d_jobs, uint32_t n_jobs, uint32_t total_blocks, long long* d_mm, unsigned long long* d_bsum,
                                cudaStream_t st);
cudaError_t launch_narrow(const NarrowJob* d_jobs, uint32_t n_jobs, uint32_t total_blocks, const unsigned long long* d_bsum, cudaStream_t st);
// Non-dictionary string pages -> chunk-local dictionary indices (intern_strings.cu): rebuild the DELTA_BYTE_ARRAY
// values, hash and insert every value into its chunk's table, rank each chunk's used slots (first occurrences to the
// host, counts per chunk), copy the distinct rebuilt values to the host, then pack every page's indices into its hole
constexpr uint32_t kFrontSeg = 1024;  // values of one StrFrontJob
cudaError_t launch_str_unfront(const StrChunk* d_chunks, const StrFrontJob* d_jobs, uint32_t n_jobs, cudaStream_t st);
cudaError_t launch_str_hash(const StrChunk* d_chunks, uint32_t n_chunks, uint32_t total_values, cudaStream_t st);
cudaError_t launch_str_compact(const StrChunk* d_chunks, uint32_t n_chunks, uint32_t total_slots, uint32_t* d_counts, cudaStream_t st);
cudaError_t launch_str_gather(const StrChunk* d_chunks, uint32_t n_chunks, uint32_t total_slots, cudaStream_t st);
cudaError_t launch_str_codes(const StrCodeJob* d_jobs, uint32_t n_jobs, uint32_t total_groups, cudaStream_t st);
// DELTA_BINARY_PACKED int64 pages -> dense values (delta_int64.cu): three launches per upload whatever its pages.
// `scratch`: dbp_scratch_bytes(n_groups) bytes, 8-byte aligned
size_t dbp_scratch_bytes(uint32_t n_groups);
cudaError_t launch_dbp_decode(const uint8_t* stage, const DbpPage* d_pages, uint32_t n_pages, const DbpMini* d_mbs, uint32_t n_groups,
                              void* scratch, cudaStream_t st);
// LZ4_RAW PLAIN int64 / double pages -> dense values (lz4_pages.cu): one launch per upload, one warp per page.
cudaError_t launch_lz4_pages(const uint8_t* stage, const Lz4Job* d_jobs, uint32_t n_jobs, cudaStream_t st);
// partial-table exchange over peer-mapped mailboxes (comm.cu)
cudaError_t launch_comm_push(const CommPush& p, int sm_count, cudaStream_t st);
cudaError_t launch_comm_wait(const CommWait& w, cudaStream_t st);
cudaError_t launch_merge_dense(const QueryDesc& q, const CommMerge& m, cudaStream_t st);
cudaError_t launch_rows(const QueryDesc* d_q, const QueryDesc& q, int sm_count, cudaStream_t st);
cudaError_t launch_finalize(const FinalizeDesc& f, cudaStream_t st);
cudaError_t launch_merge(const QueryDesc& q, const void* partial, size_t src_slots, cudaStream_t st);
cudaError_t launch_finalize_dense(const DenseOut& f, cudaStream_t st);
cudaError_t launch_gather_pages(const void* stage, void* image, const PageCopy* table, uint32_t n, cudaStream_t st);
cudaError_t launch_make_seeds(void* image, uint64_t jobs_off, uint32_t n_jobs, uint32_t max_chunks, cudaStream_t st);
cudaError_t launch_decode(const ChunkDesc& c, int32_t* out_i32, long long* out_i64, uint8_t* out_valid, int sm_count,
                          cudaStream_t st);

}  // namespace fgpu
