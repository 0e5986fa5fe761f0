// The host half of result export: the shape of a result's Arrow columns, and the columns whose layout is decided on the
// host (dictionary keys, validity from per-row bytes, dictionaries).  The device half (launches, copies back,
// synchronisations) stays with each result path in engine.cpp.
#pragma once
#include <algorithm>
#include <cstdint>
#include <memory>
#include <string>
#include <vector>

#include "arrow_export.h"

namespace fgpu {

struct GlobalDict;

struct KeyOut {
  std::string name;
  bool is_int64 = false;
  bool is_float = false;
  bool is_bool = false;  // boolean Distinct key: no dictionary, never NULL
  const GlobalDict* dict = nullptr;
  std::vector<std::string> dict_snapshot;  // values by id at execute time
};

// A result's columns: the keys with their dictionaries snapshotted at execute time (the plan may be reused while they
// grow), then the aggregates' names and types.
struct ResultShape {
  std::vector<KeyOut> keys;
  std::vector<std::string> agg_names;
  std::vector<uint8_t> agg_is_float;
};

// A utf8 dictionary column of the entries `ids` of `values` (all of them when null), in that order.
std::unique_ptr<OwnedColumn> dict_column(const std::vector<std::string>& values, const std::vector<uint32_t>* ids);

// Which dictionary a key column exports: the values its rows use, in increasing id order, or every value.
enum class KeyDict { kUsed, kWhole };

// Per-row ids as the kernels write them, mapped to "id, or NULL" in one place.
constexpr uint32_t kNullId = 0xffffffffu;
inline uint32_t row_id(uint32_t v) { return v; }
inline uint32_t row_id(int32_t v) { return v < 0 ? kNullId : uint32_t(v); }
inline uint32_t row_id(long long v) { return v == 0 ? kNullId : uint32_t(v - 1); }

// Makes `col` a dictionary key column (format "I") of n rows from the per-row ids a kernel wrote: uint32 with
// 0xffffffff for NULL (k_finalize_dense), int32 with -1 (k_rows, the decode kernel), or int64 id + 1 with 0
// (k_finalize).  The indices go to `out`, which may be `ids` itself, or to col.data when `out` is null; a NULL row gets
// index 0.  A whole dictionary is a copy of `prepared` when one is given.  A validity bitmap is written exactly when a
// row is NULL.  may_null == false promises that none is: indices written in place into a whole dictionary then cost no
// pass over the rows.
template <class T>
void dict_key_column(OwnedColumn& col, const T* ids, size_t n, uint32_t* out, const std::vector<std::string>& values, KeyDict which,
                     const OwnedColumn* prepared = nullptr, bool may_null = true) {
  col.format = "I";  // dictionary<uint32, binary>
  if (!out) {
    col.data.resize(n * 4);
    out = reinterpret_cast<uint32_t*>(col.data.data());
  }
  std::vector<uint32_t> remap, used;
  bool any_null = may_null;
  if (which == KeyDict::kUsed) {  // used ids in increasing order -> dense indices (O(rows + cardinality))
    remap.assign(values.size(), 0);
    any_null = false;
    for (size_t i = 0; i < n; i++) {
      const uint32_t id = row_id(ids[i]);
      if (id == kNullId) any_null = true;
      else remap[id] = 1;
    }
    for (size_t g = 0; g < remap.size(); g++)
      if (remap[g]) {
        remap[g] = uint32_t(used.size());
        used.push_back(uint32_t(g));
      }
  }
  if (any_null) col.validity.assign((n + 7) / 8, 0);
  if (any_null || which == KeyDict::kUsed || static_cast<const void*>(ids) != out) {
    for (size_t i = 0; i < n; i++) {
      const uint32_t id = row_id(ids[i]);
      if (id == kNullId) {
        out[i] = 0;
        col.null_count++;
        continue;
      }
      out[i] = which == KeyDict::kUsed ? remap[id] : id;
      if (any_null) set_bit(col.validity, int64_t(i));
    }
  }
  if (col.null_count == 0) col.validity.clear();
  if (which == KeyDict::kUsed) {
    col.dictionary = dict_column(values, &used);
  } else if (prepared) {
    col.dictionary = std::make_unique<OwnedColumn>();
    col.dictionary->format = prepared->format;
    col.dictionary->length = prepared->length;
    col.dictionary->data = prepared->data;
    col.dictionary->offsets = prepared->offsets;
  } else {
    col.dictionary = dict_column(values, nullptr);
  }
}

// Makes `col` a boolean key column (format "b") of n rows from the per-row ids a kernel wrote for a two-entry code key
// (id 0 false, 1 true; see row_id), bit-packed in place over `ids`: byte j is written once ids[8j .. 8j+7] are read, and
// it never lies past them.  A boolean key is never NULL (project.go:397-467 builds it without validity).
template <class T>
void bool_key_column(OwnedColumn& col, T* ids, size_t n) {
  col.format = "b";
  uint8_t* bits = reinterpret_cast<uint8_t*>(ids);
  for (size_t j = 0; j * 8 < n; j++) {
    uint8_t b = 0;
    for (size_t i = j * 8; i < std::min(n, j * 8 + 8); i++) b |= uint8_t(row_id(ids[i]) == 1) << (i & 7);
    bits[j] = b;
  }
}

// The validity of n rows from one byte per row (0: NULL), as the kernels write it: a bitmap exactly when a row is NULL.
void validity_from_bytes(OwnedColumn& col, const uint8_t* valid, size_t n);

// Writes `values` as [u32 length][bytes]... into buf (when buf is not null) and reports its length and count; false when
// cap is too small for it.  fgpu_dict_preload reads the same blob.
bool write_dict_blob(const std::vector<std::string>& values, uint8_t* buf, uint64_t cap, uint64_t* out_len, uint32_t* out_count);

}  // namespace fgpu
