// Column residency: the host images of a part's columns go to the device, and the images the scan kernels derive from
// resident columns are built on first use.
#pragma once
#include <cstdint>
#include <string>
#include <utility>
#include <vector>

#include "context.h"

namespace fgpu {

// What making columns resident cost.  h2d_bytes counts the meta regions, the transfers of PLAIN value regions,
// DELTA_BINARY_PACKED streams and LZ4_RAW blocks, the DELTA_BINARY_PACKED page and miniblock tables and the LZ4_RAW job
// tables; build_us is the host's page walk and string interning, enqueue_us the host's time queueing the uploads.
struct UploadStats {
  uint64_t h2d_bytes = 0;
  double build_us = 0, enqueue_us = 0;
};

// Makes the listed columns resident, in list order, on the engine stream: one intern batch over the columns already
// walked but not built, then each column walked and uploaded if it is built, then one intern batch over the columns
// that were not and their uploads.  refuse_unreadable: a column with an unreadable chunk fails with
// FGPU_ERR_UNSUPPORTED and nothing after it is uploaded; otherwise such a column is skipped.  The caller synchronises
// the stream before release_staging.
int32_t upload_columns(fgpu_ctx* ctx, Table* table, const std::vector<std::pair<Part*, std::string>>& cols, UploadStats* st,
                       bool refuse_unreadable);

// Every column of a part being put: host images built in parallel, uploaded, the stream synchronised and the staging
// released.  On error the part's device memory is freed.
int32_t upload_part(fgpu_ctx* ctx, Table* table, Part* part);

// Flat code arrays of one dictionary column of a part (every row group, one allocation), derived on the device
// from the resident hybrid image the first time the tile-aggregate kernel needs the column (k_flatten).
int32_t ensure_flat(fgpu_ctx* ctx, Part* part, const std::string& column);

// Frame-of-reference and prefix-sum images of resident INT64 columns for the sorted-run kernel (see residency.cpp).
int32_t ensure_narrow(fgpu_ctx* ctx, const std::vector<std::pair<Part*, std::string>>& want,
                      const std::vector<std::pair<Part*, std::string>>& want_prefix);

// After the stream has been synchronised the host staging of uploaded columns can go.
void release_staging(fgpu_ctx* ctx);

void free_part(fgpu_ctx* ctx, Part* p);

}  // namespace fgpu
