#include "result.h"

#include <cstring>

namespace fgpu {

std::unique_ptr<OwnedColumn> dict_column(const std::vector<std::string>& values, const std::vector<uint32_t>* ids) {
  auto d = std::make_unique<OwnedColumn>();
  d->format = "z";
  d->length = int64_t(ids ? ids->size() : values.size());
  d->offsets.push_back(0);
  for (size_t i = 0; i < size_t(d->length); i++) {
    const std::string& v = values[ids ? (*ids)[i] : i];
    d->data.insert(d->data.end(), v.begin(), v.end());
    d->offsets.push_back(int32_t(d->data.size()));
  }
  return d;
}

void validity_from_bytes(OwnedColumn& col, const uint8_t* valid, size_t n) {
  size_t nulls = 0;
  for (size_t i = 0; i < n; i++) nulls += valid[i] ? 0 : 1;
  if (!nulls) return;
  col.validity.assign((n + 7) / 8, 0);
  for (size_t i = 0; i < n; i++)
    if (valid[i]) set_bit(col.validity, int64_t(i));
  col.null_count = int64_t(nulls);
}

bool write_dict_blob(const std::vector<std::string>& values, uint8_t* buf, uint64_t cap, uint64_t* out_len, uint32_t* out_count) {
  uint64_t need = 0;
  for (const std::string& v : values) need += 4 + v.size();
  *out_len = need;
  *out_count = uint32_t(values.size());
  if (!buf) return true;
  if (cap < need) return false;
  for (const std::string& v : values) {
    const uint32_t l = uint32_t(v.size());
    std::memcpy(buf, &l, 4);
    std::memcpy(buf + 4, v.data(), v.size());
    buf += 4 + v.size();
  }
  return true;
}

}  // namespace fgpu
