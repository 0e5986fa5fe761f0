#include "part_store.h"

#include <algorithm>
#include <cstring>
#include <sstream>
#include <unordered_map>

namespace fgpu {
namespace {

constexpr size_t kAlign = 128;
constexpr size_t kTailPad = 16;

// Column image layout: [meta region: every section the host assembles][extent region: PLAIN value
// bytes copied verbatim from the source file].  Section offsets of the extent region are recorded
// relative to its start and rebased when the meta size is final.
struct ImageWriter {
  ImageStaging& staging;
  std::vector<uint8_t>& buf;        // staging.meta
  uint64_t ext_size = 0;
  uint64_t dev_size = 0;            // device-only region behind the extents (seeds derived on the device)
  bool device_seeds = false;
  std::vector<SeedJob> jobs;
  explicit ImageWriter(ImageStaging& s) : staging(s), buf(s.meta) {}
  uint64_t reserve_dev(uint64_t n) {
    dev_size = (dev_size + kAlign - 1) / kAlign * kAlign;
    uint64_t off = dev_size;
    dev_size += n + kTailPad;
    return off;
  }
  // queues k_make_seeds' derivation of n_chunks cursor seeds from the run directory at runs_off (val0_off: the chunks'
  // first value ordinals, ~0: chunk * 128); returns the seeds' offset in the device-only region
  int64_t seed_job(int64_t runs_off, uint32_t n_runs, uint32_t total, uint32_t n_chunks, bool is_def, uint64_t val0_off) {
    SeedJob j{};
    j.runs_off = uint64_t(runs_off);
    j.seeds_off = reserve_dev(uint64_t(n_chunks) * sizeof(Seed));
    j.val0_off = val0_off;
    j.n_runs = n_runs;
    j.total = total;
    j.n_chunks = n_chunks;
    j.is_def = is_def ? 1 : 0;
    jobs.push_back(j);
    return int64_t(j.seeds_off);
  }
  size_t begin() {
    size_t n = (buf.size() + kAlign - 1) / kAlign * kAlign;
    buf.resize(n, 0);
    return n;
  }
  void append(const void* p, size_t n) {
    const uint8_t* b = static_cast<const uint8_t*>(p);
    buf.insert(buf.end(), b, b + n);
  }
  void end() { buf.resize(buf.size() + kTailPad, 0); }
  int64_t section(const void* p, size_t n) {
    size_t off = begin();
    append(p, n);
    end();
    return int64_t(off);
  }
  // reserves an aligned hole in the extent region; returns its offset inside that region
  uint64_t begin_extent() {
    ext_size = (ext_size + kAlign - 1) / kAlign * kAlign;
    return ext_size;
  }
  void add_extent(const uint8_t* src, uint64_t len) {
    if (len == 0) return;
    std::vector<Extent>& extents = staging.extents;
    if (!extents.empty() && extents.back().src + extents.back().len == src && extents.back().dst_off + extents.back().len == ext_size)
      extents.back().len += len;  // contiguous in the file too: one copy
    else
      extents.push_back({src, len, ext_size});
    ext_size += len;
  }
  // reserves the values of a page the device fills (8 * n bytes of the extent region, not copied) and queues the page
  // with its miniblocks (`mbs`: the chunk's list); its hole is relative to the extent region until finish_image rebases it
  void add_hole(const ValuePage& pg, const std::vector<DbpMiniblock>& mbs) {
    ValuePage h = pg;
    h.hole = ext_size;
    h.mb0 = uint32_t(staging.dbp_mbs.size());
    staging.dbp_mbs.insert(staging.dbp_mbs.end(), mbs.begin() + pg.mb0, mbs.begin() + pg.mb0 + pg.n_mb);
    staging.value_pages.push_back(h);
    ext_size += uint64_t(pg.n) * 8;
  }
  void end_extent() { ext_size += kTailPad; }
};

inline void or_bits(std::vector<uint64_t>& bm, uint64_t pos, uint64_t bits8) {
  size_t w = size_t(pos >> 6);
  unsigned sh = unsigned(pos & 63);
  bm[w] |= bits8 << sh;
  if (sh > 56 && w + 1 < bm.size()) bm[w + 1] |= bits8 >> (64 - sh);
}

inline void set_range(std::vector<uint64_t>& bm, uint64_t pos, uint64_t len) {
  uint64_t end = pos + len;
  while (pos < end) {
    size_t w = size_t(pos >> 6);
    unsigned sh = unsigned(pos & 63);
    uint64_t take = std::min<uint64_t>(64 - sh, end - pos);
    uint64_t mask = (take == 64) ? ~0ull : (((1ull << take) - 1ull) << sh);
    bm[w] |= mask;
    pos += take;
  }
}

inline uint64_t popcount_range(const std::vector<uint64_t>& bm, uint64_t pos, uint64_t end) {
  uint64_t n = 0;
  while (pos < end) {
    size_t w = size_t(pos >> 6);
    unsigned sh = unsigned(pos & 63);
    uint64_t take = std::min<uint64_t>(64 - sh, end - pos);
    uint64_t mask = (take == 64) ? ~0ull : (((1ull << take) - 1ull) << sh);
    n += uint64_t(__builtin_popcountll(bm[w] & mask));
    pos += take;
  }
  return n;
}

bool is_dict_encoding(int32_t e) { return e == ENC_RLE_DICTIONARY || e == ENC_PLAIN_DICTIONARY; }
bool is_delta_string(int32_t e) { return e == ENC_DELTA_LENGTH_BYTE_ARRAY || e == ENC_DELTA_BYTE_ARRAY; }

// Length prefixes of one PLAIN BYTE_ARRAY page holding `n` values: one offset per value, from the chunk's first PLAIN
// value region.  Every value must lie inside the page and the values must fill it.
bool walk_plain_strings(const PageInfo& pg, uint32_t n, ChunkWalk* wk, std::string* err) {
  if (!wk->str_base) wk->str_base = pg.values;
  const uint64_t base = uint64_t(pg.values - wk->str_base);  // pages are walked in file order
  if (base + pg.values_len > 0xffffffffull) { *err = "PLAIN string pages of one chunk span more than 4 GiB"; return false; }
  const uint8_t* q = pg.values;
  const uint8_t* end = pg.values + pg.values_len;
  const bool start_len = !wk->str_len.empty();  // the chunk holds delta pages too: values are addressed by start and length
  for (uint32_t i = 0; i < n; i++) {
    if (end - q < 4) { *err = "PLAIN string page shorter than its value count"; return false; }
    uint32_t l;
    std::memcpy(&l, q, 4);
    if (l > uint64_t(end - q) - 4) { *err = "PLAIN string length prefix overruns its page"; return false; }
    wk->str_off.push_back(uint32_t(base + uint64_t(q - pg.values) + (start_len ? 4 : 0)));
    if (start_len) wk->str_len.push_back(l);
    q += 4 + uint64_t(l);
  }
  if (q != end) { *err = "PLAIN string page holds more values than its definition levels"; return false; }
  wk->str_span = uint32_t(base + pg.values_len);
  return true;
}

// Values of one DELTA_LENGTH_BYTE_ARRAY (all lengths, then all bytes) or DELTA_BYTE_ARRAY (all prefix lengths, all
// suffix lengths, then all suffix bytes) page holding `n` values.  The lengths must be non-negative and their bytes
// must fill the page exactly; a prefix may not be longer than the value before it ("" at the start of the page).
// DELTA_LENGTH_BYTE_ARRAY values are addressed in the file bytes, DELTA_BYTE_ARRAY values in the rebuilt region
// (offsets relative to its start until the walk of the chunk ends).
bool walk_delta_strings(const PageInfo& pg, uint32_t n, ChunkWalk* wk, std::string* err) {
  const bool dba = pg.encoding == ENC_DELTA_BYTE_ARRAY;
  const std::string what = dba ? "DELTA_BYTE_ARRAY" : "DELTA_LENGTH_BYTE_ARRAY";
  if (!wk->str_base) wk->str_base = pg.values;
  const uint64_t base = uint64_t(pg.values - wk->str_base);
  if (base + pg.values_len > 0xffffffffull) { *err = what + " pages of one chunk span more than 4 GiB"; return false; }
  if (wk->str_len.empty() && !wk->str_off.empty()) {  // PLAIN values walked so far: to start and length
    for (uint32_t& o : wk->str_off) {
      uint32_t l;
      std::memcpy(&l, wk->str_base + o, 4);
      wk->str_len.push_back(l);
      o += 4;
    }
  }
  const uint8_t* q = pg.values;
  const uint8_t* const end = pg.values + pg.values_len;
  std::vector<int32_t> a, b;
  uint64_t used = 0;
  std::string e;
  if (!decode_delta_binary_packed(q, uint64_t(end - q), n, &a, &used, &e)) {
    *err = what + (dba ? " prefix lengths: " : " lengths: ") + e;
    return false;
  }
  q += used;
  if (dba) {
    if (!decode_delta_binary_packed(q, uint64_t(end - q), n, &b, &used, &e)) { *err = what + " suffix lengths: " + e; return false; }
    q += used;
  }
  const std::vector<int32_t>& lens = dba ? b : a;
  uint64_t total = 0, prev = 0;
  for (uint32_t i = 0; i < n; i++) {
    if (lens[i] < 0) { *err = what + (dba ? " suffix length is negative" : " length is negative"); return false; }
    if (dba) {
      if (a[i] < 0) { *err = what + " prefix length is negative"; return false; }
      if (uint64_t(a[i]) > prev) { *err = what + " prefix is longer than the value before it"; return false; }
      prev = uint64_t(a[i]) + uint64_t(b[i]);
    }
    total += uint64_t(lens[i]);
  }
  if (total != uint64_t(end - q)) {
    *err = what + (dba ? " suffix lengths do not add up to the page's value bytes" : " lengths do not add up to the page's value bytes");
    return false;
  }
  uint64_t pos = base + uint64_t(q - pg.values);  // file offset of the first value's (suffix) bytes
  if (!dba) {
    for (uint32_t i = 0; i < n; i++) {
      wk->str_off.push_back(uint32_t(pos));
      wk->str_len.push_back(uint32_t(a[i]));
      pos += uint64_t(a[i]);
    }
  } else {
    const StrFront f{uint32_t(wk->str_off.size()), uint32_t(wk->str_pre.size()), uint32_t(wk->str_wmin.size()), n};
    uint64_t out = wk->str_rebuilt_len;
    for (uint32_t i = 0; i < n; i++) {
      const uint64_t len = uint64_t(a[i]) + uint64_t(b[i]);
      if (out + len > 0xffffffffull) { *err = "DELTA_BYTE_ARRAY values of one chunk exceed 4 GiB"; return false; }
      wk->str_off.push_back(uint32_t(out));
      wk->str_len.push_back(uint32_t(len));
      wk->str_pre.push_back(uint32_t(a[i]));
      wk->str_suf.push_back(uint32_t(pos));
      if (i % 32 == 0) wk->str_wmin.push_back(uint32_t(a[i]));
      else wk->str_wmin.back() = std::min(wk->str_wmin.back(), uint32_t(a[i]));
      out += len;
      pos += uint64_t(b[i]);
    }
    wk->str_rebuilt_len = out;
    wk->str_fronts.push_back(f);
  }
  wk->str_span = uint32_t(base + pg.values_len);
  return true;
}

// One DELTA_BINARY_PACKED page of an INT64 chunk holding `n` non-null values, the chunk's values [v0, v0 + n): parsed
// and validated, not unpacked (the host's work is per miniblock; the device unpacks at upload).
bool walk_delta_int64(const PageInfo& pg, uint32_t n, uint32_t v0, ChunkWalk* wk, std::string* err) {
  DbpStream s;
  if (!parse_delta_binary_packed<int64_t>(pg.values, pg.values_len, n, &s, err)) {
    *err = "int64 values: " + *err;
    return false;
  }
  if (n == 0) return true;
  wk->value_pages.push_back({FILL_DBP, pg.values, s.used, v0, n, int64_t(s.first), s.per_mb, uint32_t(wk->dbp_mbs.size()),
                             uint32_t(s.mbs.size())});
  for (DbpMiniblock& mb : s.mbs) {
    mb.first += v0;
    wk->dbp_mbs.push_back(mb);
  }
  return true;
}

// The entries of a chunk's string dictionary page, validated, each handed to `entry(bytes, length)`.
template <typename F>
bool each_dict_string(const ChunkMeta& cm, F entry, std::string* err) {
  const uint8_t* p = cm.dict;
  const uint8_t* end = cm.dict + cm.dict_len;
  for (uint32_t i = 0; i < cm.dict_num_values; i++) {
    if (end - p < 4) { *err = "dictionary page truncated"; return false; }
    uint32_t l;
    std::memcpy(&l, p, 4);
    p += 4;
    if (l > uint64_t(end - p)) { *err = "dictionary entry overruns page"; return false; }
    entry(p, l);
    p += l;
  }
  return true;
}

// The footer facts of one chunk: known before its pages are walked (a part's skeleton) and kept by the built chunk.
ChunkHost chunk_footer(const ChunkMeta& cm, const SchemaLeaf& leaf, uint32_t n_rows) {
  ChunkHost ch;
  ch.phys = leaf.phys;
  ch.stored_bytes = uint64_t(cm.codec != 0 ? cm.total_uncompressed_size : cm.total_compressed_size);
  ch.codec = cm.codec;
  ch.has_minmax = cm.has_minmax;
  ch.min_bits = cm.min_bits;
  ch.max_bits = cm.max_bits;
  ch.null_count = (cm.null_count < 0 && leaf.max_def == 0) ? 0 : cm.null_count;  // (a required column has none)
  ch.has_minmax_str = cm.has_minmax_str;
  ch.min_str = cm.min_str;
  ch.max_str = cm.max_str;
  ch.desc.n_rows = n_rows;
  return ch;
}

}  // namespace

void unfront_strings(ChunkWalk* wk) {
  if (wk->str_fronts.empty() || !wk->str_rebuilt_host.empty()) return;
  wk->str_rebuilt_host.resize(size_t(wk->str_rebuilt_len) + 1);
  uint8_t* const rb = wk->str_rebuilt_host.data();
  for (const StrFront& f : wk->str_fronts) {
    const uint8_t* prev = nullptr;
    for (uint32_t i = 0; i < f.n; i++) {
      uint8_t* dst = rb + (wk->str_off[f.v0 + i] - wk->str_rb0);
      const uint32_t pre = wk->str_pre[f.d0 + i];
      if (pre) std::memmove(dst, prev, pre);
      std::memcpy(dst + pre, wk->str_base + wk->str_suf[f.d0 + i], wk->str_len[f.v0 + i] - pre);
      prev = dst;
    }
  }
  wk->str_rebuilt = rb;
}

void fill_value_pages(const ImageStaging& s, uint8_t* image) {
  for (const ValuePage& pg : s.value_pages) {
    uint8_t* dst = image + pg.hole;
    if (pg.fill == FILL_DBP)
      unpack_delta_binary_packed<int64_t>(pg.src, pg.first, s.dbp_mbs.data() + pg.mb0, pg.n_mb, pg.v0, reinterpret_cast<int64_t*>(dst));
    else
      unpack_lz4_raw(pg.src, pg.len, dst, uint64_t(pg.n) * 8);
  }
}

namespace {

// Walks and validates every page of one column chunk (first half of building it).
void walk_chunk(const ChunkMeta& cm, const SchemaLeaf& leaf, uint32_t n_rows, ChunkWalk* wk) {
  ChunkHost* out = &wk->host;
  *out = chunk_footer(cm, leaf, n_rows);
  if (!cm.error.empty()) { out->error = cm.error; return; }
  if (leaf.phys != PT_INT64 && leaf.phys != PT_DOUBLE && leaf.phys != PT_BYTE_ARRAY) {
    out->error = "unsupported physical type " + std::to_string(leaf.phys);
    return;
  }
  if (leaf.is_unsigned) { out->error = "uint64 columns are not supported"; return; }
  if (leaf.max_def > 1) { out->error = "nested optional columns are not supported"; return; }
  bool any_dict = false, any_plain = false;
  for (const PageInfo& pg : cm.pages) {
    if (is_dict_encoding(pg.encoding)) any_dict = true;
    else if (pg.encoding == ENC_PLAIN || (leaf.phys == PT_BYTE_ARRAY && is_delta_string(pg.encoding)) ||
             (leaf.phys == PT_INT64 && pg.encoding == ENC_DELTA_BINARY_PACKED))
      any_plain = true;
    else { out->error = "unsupported page encoding " + std::to_string(pg.encoding); return; }
  }
  // (a string chunk may hold both: a dictionary whose writer fell back to PLAIN part of the way through)
  if (any_dict && any_plain && leaf.phys != PT_BYTE_ARRAY) { out->error = "column chunk mixes dictionary and PLAIN pages"; return; }

  // ---- definition levels --------------------------------------------------------------------
  std::string err;
  std::vector<uint8_t>& defstream = wk->defstream;
  std::vector<HostRun>& defruns = wk->defruns;
  std::vector<uint64_t>& valid = wk->valid;  // bitset, only when max_def == 1
  std::vector<uint32_t> page_nn(cm.pages.size());
  uint32_t n_values = n_rows;
  bool all_present = false;  // optional column whose definition levels are one run of 1s per page: no bitset needed
  if (leaf.max_def == 1) {
    uint32_t row = 0;
    for (size_t p = 0; p < cm.pages.size(); p++) {
      const PageInfo& pg = cm.pages[p];
      if (!walk_hybrid(pg.def, pg.def_len, 1, pg.num_values, row, uint32_t(defstream.size()), &defruns, &err)) {
        out->error = "definition levels: " + err;
        return;
      }
      defstream.insert(defstream.end(), pg.def, pg.def + pg.def_len);
      row += pg.num_values;
    }
    if (row != n_rows) { out->error = "definition levels do not cover the row group"; return; }
    all_present = defruns.size() == 1 && (defruns[0].meta & 1u) == 0 && defruns[0].val == 1;
    for (size_t p = 0; p < cm.pages.size() && all_present; p++)
      if (cm.pages[p].num_nulls > 0) {
        out->error = "page num_nulls disagrees with its definition levels";
        return;
      }
  }
  if (leaf.max_def == 1 && !all_present) {
    valid.assign((size_t(n_rows) + 63) / 64 + 1, 0);
    for (size_t k = 0; k < defruns.size(); k++) {
      const HostRun& r = defruns[k];
      uint32_t end = (k + 1 < defruns.size()) ? defruns[k + 1].start : n_rows;
      uint32_t len = end - r.start;
      if ((r.meta & 1u) == 0) {
        if (r.val) set_range(valid, r.start, len);
      } else {
        for (uint32_t done = 0; done < len; done += 8) {
          uint64_t b = defstream[r.off + done / 8];
          if (len - done < 8) b &= (1ull << (len - done)) - 1ull;
          or_bits(valid, uint64_t(r.start) + done, b);
        }
      }
    }
    uint32_t row = 0;
    uint64_t total_valid = 0;
    for (size_t p = 0; p < cm.pages.size(); p++) {
      const PageInfo& pg = cm.pages[p];
      uint64_t nn = popcount_range(valid, row, uint64_t(row) + pg.num_values);
      if (pg.num_nulls >= 0 && uint64_t(pg.num_values) - uint64_t(pg.num_nulls) != nn) {
        out->error = "page num_nulls disagrees with its definition levels";
        return;
      }
      page_nn[p] = uint32_t(nn);
      total_valid += nn;
      row += pg.num_values;
    }
    n_values = uint32_t(total_valid);
  } else {
    for (size_t p = 0; p < cm.pages.size(); p++) page_nn[p] = cm.pages[p].num_values;
  }
  wk->n_values = n_values;

  // ---- values -------------------------------------------------------------------------------
  std::vector<uint8_t>& vstream = wk->vstream;
  std::vector<HostRun>& vruns = wk->vruns;
  if (any_dict || leaf.phys == PT_BYTE_ARRAY) {
    uint32_t vo = 0;
    for (size_t p = 0; p < cm.pages.size(); p++) {
      const PageInfo& pg = cm.pages[p];
      if (page_nn[p] == 0) continue;
      if (pg.encoding == ENC_PLAIN || is_delta_string(pg.encoding)) {  // strings: one bit-packed run whose hole the section writing places here
        const uint32_t first = uint32_t(wk->str_off.size());
        const bool ok = pg.encoding == ENC_PLAIN ? walk_plain_strings(pg, page_nn[p], wk, &err) : walk_delta_strings(pg, page_nn[p], wk, &err);
        if (!ok) { out->error = err; return; }
        wk->str_pages.push_back(StrPage{uint32_t(vruns.size()), first, page_nn[p]});
        vruns.push_back(HostRun{vo, uint32_t(vstream.size()), 0, 1u});
        vo += page_nn[p];
        continue;
      }
      if (pg.values_len < 1) { out->error = "dictionary-index page without bit width"; return; }
      int bw = pg.values[0];
      if (bw > 32) { out->error = "dictionary index bit width > 32"; return; }
      if (!walk_hybrid(pg.values + 1, pg.values_len - 1, bw, page_nn[p], vo, uint32_t(vstream.size()), &vruns, &err)) {
        out->error = "dictionary indices: " + err;
        return;
      }
      vstream.insert(vstream.end(), pg.values + 1, pg.values + pg.values_len);
      vo += page_nn[p];
    }
    out->desc.kind = (leaf.phys == PT_BYTE_ARRAY) ? CK_DICT_STR : CK_DICT64;
    // the rebuilt DELTA_BYTE_ARRAY values go behind the file bytes, in the same 32-bit address space
    if (!wk->str_fronts.empty()) {
      const uint64_t rb0 = (uint64_t(wk->str_span) + 15) & ~uint64_t(15);
      if (rb0 + wk->str_rebuilt_len > 0xffffffffull) { out->error = "DELTA_BYTE_ARRAY values of one chunk exceed 4 GiB"; return; }
      wk->str_rb0 = uint32_t(rb0);
      for (const StrFront& f : wk->str_fronts)
        for (uint32_t i = f.v0; i < f.v0 + f.n; i++) wk->str_off[i] += uint32_t(rb0);
    }
  } else {
    uint32_t vo = 0;
    for (size_t p = 0; p < cm.pages.size(); p++) {
      const PageInfo& pg = cm.pages[p];
      const uint32_t n = page_nn[p];
      if (pg.encoding == ENC_DELTA_BINARY_PACKED) {  // (INT64 only: the encoding check above refuses it elsewhere)
        if (!walk_delta_int64(pg, n, vo, wk, &err)) { out->error = err; return; }
      } else if (uint64_t(n) * 8 > (pg.lz4_len ? pg.lz4_len : pg.values_len)) {
        out->error = "PLAIN page shorter than its value count";
        return;
      } else if (pg.lz4_len && n > 0) {  // (the block's values become a hole the device fills)
        wk->value_pages.push_back({FILL_LZ4, pg.values, pg.values_len, vo, n});
        out->lz4_pages++;
      } else {
        wk->value_pages.push_back({FILL_COPY, pg.values, uint64_t(n) * 8, vo, n});
      }
      vo += n;
    }
    out->desc.kind = CK_PLAIN64;
  }

  // ---- dictionary ---------------------------------------------------------------------------
  uint32_t dict_size = 0;
  if (out->desc.kind == CK_DICT_STR) {
    wk->dict_entries.reserve(cm.dict_num_values);
    auto entry = [&](const uint8_t* p, uint32_t l) { wk->dict_entries.push_back({p, l}); };
    if (!each_dict_string(cm, entry, &err)) { out->error = err; return; }
    dict_size = cm.dict_num_values;
  } else if (out->desc.kind == CK_DICT64) {
    if (uint64_t(cm.dict_num_values) * 8 > cm.dict_len) { out->error = "numeric dictionary page truncated"; return; }
    wk->dict64.resize(cm.dict_num_values);
    std::memcpy(wk->dict64.data(), cm.dict, size_t(cm.dict_num_values) * 8);
    dict_size = cm.dict_num_values;
  }
  if (out->desc.kind != CK_PLAIN64) {
    for (const HostRun& r : vruns)
      if ((r.meta & 1u) == 0 && r.val >= dict_size) { out->error = "dictionary index out of range"; return; }
    if (n_values > wk->str_off.size() && dict_size == 0) { out->error = "dictionary-encoded values without a dictionary page"; return; }
  }
}

// Packs `n` indices LSB first at `w` bits into `dst` (whole bytes of 8-value groups: ceil(n / 8) * w bytes).
void pack_bits(const uint32_t* v, uint32_t n, uint32_t w, uint8_t* dst) {
  uint64_t acc = 0;
  uint32_t bits = 0;
  for (uint32_t i = 0; i < (n + 7) / 8 * 8; i++) {
    acc |= uint64_t(i < n ? v[i] : 0u) << bits;
    bits += w;
    while (bits >= 8) {
      *dst++ = uint8_t(acc);
      acc >>= 8;
      bits -= 8;
    }
  }
}

// Writes every section of one walked column chunk into the image (second half of building it).
void write_chunk(ChunkWalk& wk, uint32_t n_rows, int tile_rows, GlobalDict* dict, bool host_intern, ImageWriter& w, ChunkHost* out) {
  *out = std::move(wk.host);
  if (!out->error.empty()) return;
  const uint32_t T = uint32_t(tile_rows);
  const uint32_t n_tiles = (n_rows + T - 1) / T;
  const uint32_t n_values = wk.n_values;
  const bool has_nulls = (n_values != n_rows);
  const std::vector<uint64_t>& valid = wk.valid;
  std::vector<uint8_t>& defstream = wk.defstream;
  std::vector<HostRun>& defruns = wk.defruns;
  std::vector<uint8_t>& vstream = wk.vstream;
  std::vector<HostRun>& vruns = wk.vruns;
  std::vector<int64_t>& dict64 = wk.dict64;

  // ---- chunk-local string dictionary: the dictionary page, then the PLAIN values not in it, in order of first occurrence ----
  uint32_t dict_size = uint32_t(dict64.size());
  if (out->desc.kind == CK_DICT_STR) {
    ChunkInterner in(dict, &out->lut_host);
    out->lut_host.reserve(wk.dict_entries.size());
    for (const auto& e : wk.dict_entries) in.entry(reinterpret_cast<const char*>(e.first), e.second);
    std::vector<uint32_t> codes;  // host: per non-dictionary value; device: per distinct one (str_firsts)
    if (host_intern) {
      unfront_strings(&wk);
      codes.reserve(wk.str_off.size());
      for (uint32_t i = 0; i < uint32_t(wk.str_off.size()); i++) {
        const std::string_view s = chunk_string(wk, i);
        codes.push_back(in.add(s.data(), s.size()));
      }
    } else {  // (the intern batch left the rebuilt bytes of the distinct DELTA_BYTE_ARRAY values in str_rebuilt)
      codes.reserve(wk.str_firsts.size());
      for (uint32_t f : wk.str_firsts) {
        const std::string_view s = chunk_string(wk, f);
        codes.push_back(in.add(s.data(), s.size()));
      }
    }
    dict_size = uint32_t(out->lut_host.size());
    if (dict_size > (1u << 24)) { out->error = "PLAIN string values need a chunk dictionary of more than 2^24 entries"; return; }
    // holes for the PLAIN pages' indices, at the stream positions their pages held
    if (!wk.str_pages.empty()) {
      uint32_t bw = 1;
      while ((uint64_t(1) << bw) < dict_size) bw++;
      wk.str_w = bw;
      std::vector<uint8_t> vs;
      uint32_t src = 0, shift = 0;
      size_t sp = 0;
      for (size_t k = 0; k < vruns.size(); k++) {
        HostRun& r = vruns[k];
        if (sp < wk.str_pages.size() && wk.str_pages[sp].run == k) {
          StrPage& pg = wk.str_pages[sp++];
          vs.insert(vs.end(), vstream.begin() + src, vstream.begin() + r.off);
          src = r.off;
          r.off = uint32_t(vs.size());
          r.meta = 1u | (bw << 8);
          pg.hole = r.off;  // relative to the section until it is written
          const uint32_t bytes = (pg.n + 7) / 8 * bw;
          vs.resize(vs.size() + bytes, 0);
          if (host_intern) pack_bits(codes.data() + pg.first, pg.n, bw, vs.data() + r.off);
          shift += bytes;
        } else if (r.meta & 1u) {
          r.off += shift;
        }
      }
      vs.insert(vs.end(), vstream.begin() + src, vstream.end());
      vstream.swap(vs);
    }
    if (!host_intern) wk.str_codes = std::move(codes);
  }

  // ---- RLE run values of string dictionaries become global ids (no LUT hop for run-length data) ----
  if (out->desc.kind == CK_DICT_STR)
    for (HostRun& r : vruns)
      if ((r.meta & 1u) == 0) r.val = out->lut_host[r.val];

  // ---- chunk seeds ------------------------------------------------------------------------------
  const uint32_t n_chunks = n_tiles;  // `tile_rows` is the seed granularity (kIndexRows)
  std::vector<uint32_t> chunk_val0((has_nulls || !w.device_seeds) ? n_chunks : 0);
  if (!has_nulls && w.device_seeds) {
    // k_make_seeds derives chunk * 128 itself
  } else if (has_nulls) {
    uint64_t acc = 0;
    for (uint32_t t = 0; t < n_chunks; t++) {
      chunk_val0[t] = uint32_t(acc);
      uint64_t b = uint64_t(t) * T, e = std::min<uint64_t>(uint64_t(n_rows), b + T);
      acc += popcount_range(valid, b, e);
    }
  } else {
    for (uint32_t t = 0; t < n_chunks; t++) chunk_val0[t] = t * T;
  }
  auto make_seeds = [&](const std::vector<HostRun>& runs, uint32_t total, bool is_def) {
    std::vector<Seed> seeds(n_chunks);
    size_t k = 0;
    for (uint32_t t = 0; t < n_chunks; t++) {
      uint32_t first = is_def ? t * T : chunk_val0[t];
      while (k + 1 < runs.size() && runs[k + 1].start <= first) k++;
      Seed sd{};
      sd.val0 = chunk_val0[t];
      if (runs.empty() || first >= total) {  // nothing left to decode from this chunk on
        sd.k = uint32_t(runs.size());
        sd.start = total;
        sd.end = 0xffffffffu;
      } else {
        const HostRun& r = runs[k];
        sd.k = uint32_t(k);
        sd.start = r.start;
        sd.end = (k + 1 < runs.size()) ? runs[k + 1].start : total;
        sd.off = r.off;
        sd.val = r.val;
        sd.meta = r.meta;
      }
      seeds[t] = sd;
    }
    return seeds;
  };

  // ---- write sections ----------------------------------------------------------------------------
  const size_t before = w.buf.size();
  out->desc.has_nulls = has_nulls ? 1 : 0;
  out->desc.n_values = n_values;
  out->desc.dict_size = dict_size;
  if (out->desc.kind == CK_PLAIN64) {
    // value regions go to the device straight from the file: negative offsets mark "extent region"
    // (a page the device fills is a hole where its PLAIN twin's values would be copied to)
    const uint64_t eoff = w.begin_extent();
    for (const ValuePage& pg : wk.value_pages) {
      if (pg.fill == FILL_COPY) w.add_extent(pg.src, pg.len);
      else w.add_hole(pg, wk.dbp_mbs);
    }
    w.end_extent();
    out->off_values = -int64_t(eoff) - 1;
  } else {
    out->off_values = w.section(vstream.data(), vstream.size());
    for (StrPage& pg : wk.str_pages) pg.hole += uint64_t(out->off_values);
  }
  uint64_t val0_off = ~0ull;
  if (w.device_seeds && has_nulls) val0_off = uint64_t(w.section(chunk_val0.data(), chunk_val0.size() * 4));
  // ---- row-space directory of a nullable dictionary column whose two streams are run-length only ----
  // (what a sorted part leaves: NULLs first, then one run per value).  The sorted-run kernel walks it like
  // the directory of a column without NULLs; 0xffffffff stands for NULL (contributes 0 to the dense slot).
  std::vector<HostRun> row_runs;
  if (out->desc.kind == CK_DICT_STR && has_nulls) {
    bool rle_only = true;
    for (const HostRun& r : vruns) rle_only = rle_only && (r.meta & 1u) == 0;
    for (const HostRun& r : defruns) rle_only = rle_only && (r.meta & 1u) == 0;
    if (rle_only) {
      auto push = [&](uint32_t start, uint32_t val) {
        if (!row_runs.empty() && row_runs.back().val == val) return;
        row_runs.push_back(HostRun{start, 0, val, 0});
      };
      size_t vk = 0;
      uint32_t vord = 0;  // ordinal of the next non-null value
      for (size_t k = 0; k < defruns.size(); k++) {
        const uint32_t s0 = defruns[k].start, e0 = (k + 1 < defruns.size()) ? defruns[k + 1].start : n_rows;
        if (defruns[k].val == 0) { push(s0, 0xffffffffu); continue; }
        uint32_t row = s0;
        while (row < e0) {
          while (vk + 1 < vruns.size() && vruns[vk + 1].start <= vord) vk++;
          const uint32_t vend = (vk + 1 < vruns.size()) ? vruns[vk + 1].start : n_values;
          const uint32_t take = std::min(e0 - row, vend - vord);
          push(row, vruns[vk].val);
          row += take;
          vord += take;
        }
      }
    }
  }
  if (out->desc.kind != CK_PLAIN64) {
    out->desc.n_runs = uint32_t(vruns.size());
    uint32_t bp = 0;
    for (const HostRun& r : vruns) bp += (r.meta & 1u);
    out->desc.n_bp_runs = bp;
    std::vector<Seed> seeds;
    if (!w.device_seeds) seeds = make_seeds(vruns, n_values, false);
    HostRun sentinel{n_values, 0, 0, 0};
    vruns.push_back(sentinel);
    out->off_runs = w.section(vruns.data(), vruns.size() * sizeof(HostRun));
    if (w.device_seeds) out->dev_seeds = w.seed_job(out->off_runs, out->desc.n_runs, n_values, n_chunks, false, val0_off);
    else out->off_seeds = w.section(seeds.data(), seeds.size() * sizeof(Seed));
  }
  if (has_nulls) {
    out->desc.n_defruns = uint32_t(defruns.size());
    std::vector<Seed> seeds;
    if (!w.device_seeds) seeds = make_seeds(defruns, n_rows, true);
    HostRun sentinel{n_rows, 0, 0, 0};
    defruns.push_back(sentinel);
    out->off_def = w.section(defstream.data(), defstream.size());
    out->off_def_runs = w.section(defruns.data(), defruns.size() * sizeof(HostRun));
    if (w.device_seeds) out->dev_def_seeds = w.seed_job(out->off_def_runs, out->desc.n_defruns, n_rows, n_chunks, true, val0_off);
    else out->off_def_seeds = w.section(seeds.data(), seeds.size() * sizeof(Seed));
  }
  if (!row_runs.empty()) {
    out->desc.n_row_runs = uint32_t(row_runs.size());
    std::vector<Seed> seeds;
    if (!w.device_seeds) seeds = make_seeds(row_runs, n_rows, true);
    row_runs.push_back(HostRun{n_rows, 0, 0, 0});
    out->off_row_runs = w.section(row_runs.data(), row_runs.size() * sizeof(HostRun));
    if (w.device_seeds) out->dev_row_seeds = w.seed_job(out->off_row_runs, out->desc.n_row_runs, n_rows, n_chunks, true, ~0ull);
    else out->off_row_seeds = w.section(seeds.data(), seeds.size() * sizeof(Seed));
  }
  // Bit-packed indices are not range-checked row by row (neither here nor in the kernels): the tables they index are
  // padded to 2^w entries instead (w = widest bit-packed run of the chunk), so that any w-bit pattern of a corrupt
  // chunk reads a valid entry (dictionary entry 0) instead of memory behind the table.
  uint32_t max_w = 0;
  for (const HostRun& r : vruns)
    if (r.meta & 1u) max_w = std::max<uint32_t>(max_w, (r.meta >> 8) & 0xffu);
  const size_t padded = max_w > 0 && max_w <= 24 ? (size_t(1) << max_w) : 0;
  if (max_w > 24 && out->desc.kind != CK_PLAIN64 && (uint64_t(1) << std::min<uint32_t>(max_w, 40)) > uint64_t(dict_size) * 2 + 2) {
    out->error = "bit-packed dictionary indices wider than the dictionary";
    return;
  }
  if (out->desc.kind == CK_DICT_STR) {
    if (padded > out->lut_host.size()) {
      std::vector<uint32_t> lut = out->lut_host;
      lut.resize(padded, lut.empty() ? 0u : lut[0]);
      out->off_lut = w.section(lut.data(), lut.size() * 4);
    } else {
      out->off_lut = w.section(out->lut_host.data(), out->lut_host.size() * 4);
    }
  }
  if (out->desc.kind == CK_DICT64) {
    if (padded > dict64.size()) dict64.resize(padded, dict64.empty() ? 0 : dict64[0]);
    out->off_dict64 = w.section(dict64.data(), dict64.size() * 8);
  }
  const size_t payload = vstream.size() + (has_nulls ? defstream.size() : 0);
  out->meta_bytes = (w.buf.size() - before) - std::min(w.buf.size() - before, payload);
  if (out->dev_seeds >= 0) out->meta_bytes += uint64_t(n_chunks) * sizeof(Seed);
  if (out->dev_def_seeds >= 0) out->meta_bytes += uint64_t(n_chunks) * sizeof(Seed);
}

// Closes a column image: seed jobs table, final offsets of the extent and device-only regions.
void finish_image(ImageWriter& w, ColumnImage& img, Part* part, const std::string& column) {
  if (!w.jobs.empty()) {
    img.seed_jobs_off = uint64_t(w.section(w.jobs.data(), w.jobs.size() * sizeof(SeedJob)));
    img.n_seed_jobs = uint32_t(w.jobs.size());
    for (const SeedJob& j : w.jobs) img.max_seed_chunks = std::max(img.max_seed_chunks, j.n_chunks);
  }
  if (img.staging.meta.empty()) img.staging.meta.resize(kAlign, 0);
  // rebase extent offsets behind the (128-aligned) meta region, the device-only region behind the extents
  const uint64_t meta_size = (img.staging.meta.size() + kAlign - 1) / kAlign * kAlign;
  const uint64_t dev_base = (meta_size + w.ext_size + kAlign - 1) / kAlign * kAlign;
  for (Extent& e : img.staging.extents) e.dst_off += meta_size;
  for (ValuePage& pg : img.staging.value_pages) pg.hole += meta_size;
  for (RowGroupHost& h : part->rgs) {
    ChunkHost& ch = h.cols[column];
    if (ch.off_values < 0) ch.off_values = int64_t(meta_size) + (-ch.off_values - 1);
    if (ch.dev_seeds >= 0) ch.off_seeds = int64_t(dev_base) + ch.dev_seeds;
    if (ch.dev_def_seeds >= 0) ch.off_def_seeds = int64_t(dev_base) + ch.dev_def_seeds;
    if (ch.dev_row_seeds >= 0) ch.off_row_seeds = int64_t(dev_base) + ch.dev_row_seeds;
  }
  for (uint32_t i = 0; i < img.n_seed_jobs; i++) {
    SeedJob* j = reinterpret_cast<SeedJob*>(img.staging.meta.data() + img.seed_jobs_off) + i;
    j->seeds_off += dev_base;
  }
  img.dev_bytes = dev_base + w.dev_size + kAlign;
}


}  // namespace

bool open_part(const uint8_t* file, uint64_t len, Part* part, std::string* err) {
  if (!parse_parquet(file, len, &part->pf, err, /*walk_pages=*/false)) return false;  // page headers: on demand, per column
  part->file = file;
  part->file_bytes = len;
  part->columns.clear();
  for (const SchemaLeaf& l : part->pf.leaves) part->columns.push_back(l.name);
  for (const RowGroupMeta& rg : part->pf.row_groups) {
    if (rg.num_rows == 0) continue;
    if (rg.num_rows > 0x7fffffffll) { *err = "row group with more than 2^31 rows"; return false; }
    RowGroupHost h;
    h.n_rows = uint32_t(rg.num_rows);
    for (size_t c = 0; c < rg.chunks.size(); c++) {
      ChunkHost ch = chunk_footer(rg.chunks[c], part->pf.leaves[c], h.n_rows);  // skeleton until the column is built
      // (parquet-go sizes the filter by the chunk's values, 10 bits each: anything beyond a few MB is left alone)
      if (rg.chunks[c].bloom && rg.chunks[c].bloom_bytes <= (8u << 20))
        ch.bloom.assign(rg.chunks[c].bloom, rg.chunks[c].bloom + rg.chunks[c].bloom_bytes);
      h.cols.emplace(part->pf.leaves[c].name, std::move(ch));
    }
    part->rgs.push_back(std::move(h));
  }
  return true;
}

void walk_column(int index_rows, Table* table, Part* part, const std::string& column, bool device_seeds) {
  ColumnImage& img = part->images[column];
  if (img.built || img.walked) return;
  img.walked = true;
  img.device_seeds = device_seeds;
  size_t leaf = part->pf.leaves.size();
  for (size_t c = 0; c < part->pf.leaves.size(); c++)
    if (part->pf.leaves[c].name == column) leaf = c;
  if (leaf == part->pf.leaves.size()) {
    img.error = "column not in part";
    img.built = true;
    return;
  }
  const SchemaLeaf& sl = part->pf.leaves[leaf];
  img.walks.resize(part->rgs.size());
  bool plain_strings = false;
  size_t g = 0;
  for (RowGroupMeta& rg : part->pf.row_groups) {
    if (rg.num_rows == 0) continue;
    ChunkWalk& wk = img.walks[g];
    walk_chunk_pages(part->file, part->file_bytes, sl, rg.num_rows, &rg.chunks[leaf]);  // first touch of this chunk
    walk_chunk(rg.chunks[leaf], sl, part->rgs[g].n_rows, &wk);
    if (!wk.host.error.empty() && img.error.empty()) img.error = wk.host.error;
    plain_strings = plain_strings || (wk.host.error.empty() && !wk.str_off.empty());
    g++;
  }
  if (!plain_strings || !img.error.empty()) {
    finish_column(index_rows, table, part, column, /*host_intern=*/true);
    img.walks.clear();
  }
}

void finish_column(int index_rows, Table* table, Part* part, const std::string& column, bool host_intern) {
  ColumnImage& img = part->images[column];
  if (img.built) return;
  img.built = true;
  GlobalDict* dict = nullptr;
  for (const SchemaLeaf& l : part->pf.leaves)
    if (l.name == column && l.phys == PT_BYTE_ARRAY) dict = &table->dicts[column];
  ImageWriter w(img.staging);
  w.device_seeds = img.device_seeds;
  for (size_t g = 0; g < part->rgs.size(); g++) {
    RowGroupHost& h = part->rgs[g];
    ChunkHost ch;
    write_chunk(img.walks[g], h.n_rows, index_rows, dict, host_intern, w, &ch);
    if (!ch.error.empty() && img.error.empty()) img.error = ch.error;
    ch.bloom = std::move(h.cols[column].bloom);  // (footer-level fact of the skeleton the built chunk replaces)
    h.cols[column] = std::move(ch);
  }
  finish_image(w, img, part, column);
}

void build_column(int index_rows, Table* table, Part* part, const std::string& column, bool device_seeds) {
  walk_column(index_rows, table, part, column, device_seeds);
  ColumnImage& img = part->images[column];
  if (img.built) return;
  finish_column(index_rows, table, part, column, /*host_intern=*/true);
  img.walks.clear();
}

namespace {

inline bool bit_at(const uint8_t* bm, int64_t i) { return (bm[i >> 3] >> (i & 7)) & 1; }

// Integer view of an Arrow index buffer element.
inline int64_t arrow_index(const void* buf, char fmt, int64_t i) {
  switch (fmt) {
    case 'c': return static_cast<const int8_t*>(buf)[i];
    case 'C': return static_cast<const uint8_t*>(buf)[i];
    case 's': return static_cast<const int16_t*>(buf)[i];
    case 'S': return static_cast<const uint16_t*>(buf)[i];
    case 'i': return static_cast<const int32_t*>(buf)[i];
    case 'I': return static_cast<const uint32_t*>(buf)[i];
    case 'l': return static_cast<const int64_t*>(buf)[i];
    default: return int64_t(static_cast<const uint64_t*>(buf)[i]);
  }
}

// One Arrow column -> one column image (one chunk).
bool build_arrow_column(Table* table, Part* part, const std::string& name, const ::ArrowSchema* cs, const ::ArrowArray* ca,
                        uint32_t n_rows, std::string* err) {
  const std::string fmt = cs->format ? cs->format : "";
  const bool is_dict = cs->dictionary != nullptr;
  const bool is_i64 = !is_dict && fmt == "l";
  const bool is_f64 = !is_dict && fmt == "g";
  const bool is_str = !is_dict && (fmt == "u" || fmt == "z");
  if (!is_dict && !is_i64 && !is_f64 && !is_str) { *err = "column " + name + ": unsupported Arrow type '" + fmt + "'"; return false; }
  if (is_dict && (fmt.size() != 1 || std::string("cCsSiIlL").find(fmt[0]) == std::string::npos)) {
    *err = "column " + name + ": unsupported dictionary index type '" + fmt + "'";
    return false;
  }
  if (uint64_t(ca->length) != n_rows) { *err = "column " + name + ": length differs from the record"; return false; }
  const int64_t off = ca->offset;
  const uint8_t* validity = (ca->n_buffers > 0 && ca->null_count != 0) ? static_cast<const uint8_t*>(ca->buffers[0]) : nullptr;
  auto valid_at = [&](int64_t i) { return !validity || bit_at(validity, off + i); };

  ColumnImage& img = part->images[name];
  img.built = true;
  ImageWriter w(img.staging);
  w.device_seeds = true;
  ChunkHost ch;
  ch.desc.n_rows = n_rows;
  const uint32_t T = 128;  // seed granularity (kIndexRows)
  const uint32_t n_chunks = (n_rows + T - 1) / T;

  // ---- validity -> definition levels (the Arrow bitmap is the bit-packed level stream, LSB first) ----
  uint32_t n_values = 0;
  std::vector<uint8_t> defbits((size_t(n_rows) + 7) / 8 + 8, 0);
  std::vector<uint32_t> val0(n_chunks);
  for (uint32_t i = 0; i < n_rows; i++) {
    if (i % T == 0) val0[i / T] = n_values;
    if (valid_at(i)) {
      defbits[i >> 3] |= uint8_t(1u << (i & 7));
      n_values++;
    }
  }
  const bool has_nulls = n_values != n_rows;
  ch.null_count = int64_t(n_rows) - int64_t(n_values);
  ch.desc.has_nulls = has_nulls ? 1 : 0;
  ch.desc.n_values = n_values;

  uint64_t val0_off = ~0ull;
  if (has_nulls) val0_off = uint64_t(w.section(val0.data(), val0.size() * 4));

  if (is_i64 || is_f64) {
    ch.phys = is_i64 ? PT_INT64 : PT_DOUBLE;
    ch.desc.kind = CK_PLAIN64;
    const int64_t* src = static_cast<const int64_t*>(ca->buffers[1]) + off;
    std::vector<int64_t> packed;
    const int64_t* vals = src;
    if (has_nulls) {
      packed.reserve(n_values);
      for (uint32_t i = 0; i < n_rows; i++)
        if (valid_at(i)) packed.push_back(src[i]);
      vals = packed.data();
    }
    if (is_i64 && n_values > 0) {  // bounds for row-group pruning, as a Parquet writer would record them
      int64_t mn = vals[0], mx = vals[0];
      for (uint32_t i = 1; i < n_values; i++) { mn = std::min(mn, vals[i]); mx = std::max(mx, vals[i]); }
      ch.has_minmax = true;
      ch.min_bits = mn;
      ch.max_bits = mx;
    }
    ch.off_values = w.section(vals, size_t(n_values) * 8);
    ch.stored_bytes = uint64_t(n_values) * 8 + (has_nulls ? (n_rows + 7) / 8 : 0);
  } else {
    ch.phys = PT_BYTE_ARRAY;
    ch.desc.kind = CK_DICT_STR;
    GlobalDict* gd = &table->dicts[name];
    std::vector<uint32_t> idx;  // chunk-local index of every non-null row
    idx.reserve(n_values);
    if (is_dict) {
      const ::ArrowArray* da = ca->dictionary;
      const std::string dfmt = cs->dictionary->format ? cs->dictionary->format : "";
      if (dfmt != "u" && dfmt != "z") { *err = "column " + name + ": dictionary values must be binary/utf8, got '" + dfmt + "'"; return false; }
      const int32_t* doff = static_cast<const int32_t*>(da->buffers[1]) + da->offset;
      const char* dbytes = static_cast<const char*>(da->buffers[2]);
      ch.lut_host.reserve(size_t(da->length));
      for (int64_t i = 0; i < da->length; i++) ch.lut_host.push_back(gd->intern(dbytes ? dbytes + doff[i] : "", size_t(doff[i + 1] - doff[i])));
      for (uint32_t i = 0; i < n_rows; i++) {
        if (!valid_at(i)) continue;
        int64_t v = arrow_index(ca->buffers[1], fmt[0], off + i);
        if (v < 0 || v >= da->length) { *err = "column " + name + ": dictionary index out of range"; return false; }
        idx.push_back(uint32_t(v));
      }
    } else {
      const int32_t* soff = static_cast<const int32_t*>(ca->buffers[1]) + off;
      const char* sbytes = static_cast<const char*>(ca->buffers[2]);
      ChunkInterner in(gd, &ch.lut_host);
      for (uint32_t i = 0; i < n_rows; i++) {
        if (!valid_at(i)) continue;
        idx.push_back(in.add(sbytes ? sbytes + soff[i] : "", size_t(soff[i + 1] - soff[i])));
      }
    }
    ch.desc.dict_size = uint32_t(ch.lut_host.size());
    // index stream: raw 32-bit indices = one bit-packed run of width 32
    std::vector<HostRun> vruns;
    if (n_values > 0) vruns.push_back(HostRun{0, 0, 0, 1u | (32u << 8)});
    ch.desc.n_runs = uint32_t(vruns.size());
    ch.desc.n_bp_runs = uint32_t(vruns.size());
    vruns.push_back(HostRun{n_values, 0, 0, 0});
    ch.off_values = w.section(idx.data(), idx.size() * 4);
    ch.off_runs = w.section(vruns.data(), vruns.size() * sizeof(HostRun));
    ch.dev_seeds = w.seed_job(ch.off_runs, ch.desc.n_runs, n_values, n_chunks, false, val0_off);
    ch.off_lut = w.section(ch.lut_host.data(), ch.lut_host.size() * 4);
    ch.stored_bytes = uint64_t(n_values) * 4 + (has_nulls ? (n_rows + 7) / 8 : 0);
  }
  if (has_nulls) {
    std::vector<HostRun> druns;
    druns.push_back(HostRun{0, 0, 0, 1u | (1u << 8)});
    ch.desc.n_defruns = 1;
    druns.push_back(HostRun{n_rows, 0, 0, 0});
    ch.off_def = w.section(defbits.data(), defbits.size());
    ch.off_def_runs = w.section(druns.data(), druns.size() * sizeof(HostRun));
    ch.dev_def_seeds = w.seed_job(ch.off_def_runs, 1, n_rows, n_chunks, true, val0_off);
  }
  ch.meta_bytes = uint64_t(n_chunks) * sizeof(Seed) * ((ch.dev_seeds >= 0) + (ch.dev_def_seeds >= 0));
  part->rgs[0].cols[name] = std::move(ch);
  finish_image(w, img, part, name);
  return true;
}

}  // namespace

bool build_arrow_part(Table* table, Part* part, const ::ArrowSchema* schema, const ::ArrowArray* array, std::string* err) {
  if (!schema || !array || !schema->format || std::string(schema->format) != "+s") { *err = "Arrow part must be a struct array (record batch)"; return false; }
  if (schema->n_children != array->n_children) { *err = "Arrow schema / array children differ"; return false; }
  if (array->length < 0 || array->length > 0x7fffffffll) { *err = "record with more than 2^31 rows"; return false; }
  if (array->offset != 0 || array->null_count > 0) { *err = "sliced or nullable record structs are not supported"; return false; }
  const uint32_t n_rows = uint32_t(array->length);
  part->columns.clear();
  part->rgs.clear();
  if (n_rows == 0) return true;  // an empty record scans nothing
  RowGroupHost h;
  h.n_rows = n_rows;
  part->rgs.push_back(std::move(h));
  for (int64_t c = 0; c < schema->n_children; c++) {
    const ::ArrowSchema* cs = schema->children[c];
    const std::string name = cs->name ? cs->name : "";
    if (name.empty()) { *err = "unnamed column in Arrow part"; return false; }
    part->columns.push_back(name);
    if (!build_arrow_column(table, part, name, cs, array->children[c], n_rows, err)) return false;
  }
  return true;
}

void patch_column_pointers(Part* part, const std::string& column, const uint8_t* base) {
  for (RowGroupHost& rg : part->rgs) {
    auto it = rg.cols.find(column);
    if (it == rg.cols.end()) continue;
    ChunkHost& c = it->second;
    if (!c.error.empty()) continue;
    auto at = [&](int64_t off) -> const uint8_t* { return off < 0 ? nullptr : base + off; };
    c.desc.values = at(c.off_values);
    c.desc.runs = reinterpret_cast<const Run*>(at(c.off_runs));
    c.desc.seeds = reinterpret_cast<const Seed*>(at(c.off_seeds));
    c.desc.def = at(c.off_def);
    c.desc.def_runs = reinterpret_cast<const Run*>(at(c.off_def_runs));
    c.desc.def_seeds = reinterpret_cast<const Seed*>(at(c.off_def_seeds));
    c.desc.lut = reinterpret_cast<const uint32_t*>(at(c.off_lut));
    c.desc.dict64 = reinterpret_cast<const int64_t*>(at(c.off_dict64));
    if (c.off_row_runs >= 0) {
      c.desc.row_runs = reinterpret_cast<const Run*>(at(c.off_row_runs));
      c.desc.row_seeds = reinterpret_cast<const Seed*>(at(c.off_row_seeds));
    } else if (c.desc.kind == CK_DICT_STR && !c.desc.has_nulls && c.desc.n_bp_runs == 0) {
      c.desc.row_runs = c.desc.runs;  // no NULLs: value ordinals are rows
      c.desc.row_seeds = c.desc.seeds;
      c.desc.n_row_runs = c.desc.n_runs;
    } else {
      c.desc.row_runs = nullptr;
      c.desc.row_seeds = nullptr;
    }
  }
}

bool column_dict_values(const ParsedFile& pf, const std::string& column, GlobalDict* d, std::string* err) {
  for (size_t c = 0; c < pf.leaves.size(); c++) {
    if (pf.leaves[c].name != column) continue;
    for (const RowGroupMeta& rg : pf.row_groups) {
      const ChunkMeta& cm = rg.chunks[c];
      if (!cm.error.empty()) { *err = column + ": " + cm.error; return false; }
      bool plain_strings = false;
      for (const PageInfo& pg : cm.pages)
        plain_strings = plain_strings || (pf.leaves[c].phys == PT_BYTE_ARRAY && (pg.encoding == ENC_PLAIN || is_delta_string(pg.encoding)));
      if (plain_strings) {  // the page walk validates the dictionary page and the non-dictionary values
        ChunkWalk wk;
        walk_chunk(cm, pf.leaves[c], uint32_t(rg.num_rows), &wk);
        if (!wk.host.error.empty()) { *err = column + ": " + wk.host.error; return false; }
        unfront_strings(&wk);
        std::vector<uint32_t> lut;
        ChunkInterner in(d, &lut);
        for (const auto& e : wk.dict_entries) in.entry(reinterpret_cast<const char*>(e.first), e.second);
        for (uint32_t i = 0; i < uint32_t(wk.str_off.size()); i++) {
          const std::string_view s = chunk_string(wk, i);
          in.add(s.data(), s.size());
        }
        continue;
      }
      auto entry = [&](const uint8_t* p, uint32_t l) { d->intern(reinterpret_cast<const char*>(p), l); };
      if (!each_dict_string(cm, entry, err)) return false;
    }
  }
  return true;
}

// ---- host-only description (tests without a GPU) ---------------------------------------------------
namespace {
void json_escape(std::ostringstream& o, const std::string& s) {
  o << '"';
  for (unsigned char ch : s) {
    if (ch == '"' || ch == '\\') o << '\\' << ch;
    else if (ch < 0x20 || ch >= 0x7f) {
      char buf[8];
      snprintf(buf, sizeof buf, "\\u%04x", ch);
      o << buf;
    } else o << ch;
  }
  o << '"';
}
}  // namespace

std::string describe_part_json(const uint8_t* file, uint64_t len, int tile_rows, std::string* err) {
  Table table;
  Part part;
  if (!open_part(file, len, &part, err)) return "";
  std::vector<std::vector<uint8_t>> host_images;  // one flat host copy per column (meta + extents)
  uint64_t image_bytes = 0;
  for (const std::string& name : part.columns) {
    build_column(tile_rows, &table, &part, name);
    ColumnImage& img = part.images[name];
    std::vector<uint8_t> flat(size_t(img.dev_bytes), 0);
    std::memcpy(flat.data(), img.staging.meta.data(), img.staging.meta.size());
    for (const Extent& e : img.staging.extents) std::memcpy(flat.data() + e.dst_off, e.src, size_t(e.len));
    fill_value_pages(img.staging, flat.data());
    host_images.push_back(std::move(flat));
    patch_column_pointers(&part, name, host_images.back().data());  // pointers into the host image
    image_bytes += img.dev_bytes;
  }
  const uint32_t T = uint32_t(tile_rows);
  std::ostringstream o;
  o << "{\"image_bytes\":" << image_bytes << ",\"file_bytes\":" << len << ",\"row_groups\":[";
  for (size_t g = 0; g < part.rgs.size(); g++) {
    const RowGroupHost& rg = part.rgs[g];
    if (g) o << ',';
    o << "{\"n_rows\":" << rg.n_rows << ",\"columns\":{";
    bool firstc = true;
    for (const std::string& name : part.columns) {
      const ChunkHost& c = rg.cols.at(name);
      if (!firstc) o << ',';
      firstc = false;
      json_escape(o, name);
      o << ":{";
      if (!c.error.empty()) {
        o << "\"error\":";
        json_escape(o, c.error);
        o << '}';
        continue;
      }
      const ChunkDesc& d = c.desc;
      o << "\"kind\":" << int(d.kind) << ",\"has_nulls\":" << int(d.has_nulls) << ",\"n_values\":" << d.n_values
        << ",\"n_runs\":" << d.n_runs << ",\"n_defruns\":" << d.n_defruns << ",\"dict_size\":" << d.dict_size
        << ",\"stored_bytes\":" << c.stored_bytes << ",\"meta_bytes\":" << c.meta_bytes << ",\"null_count\":" << c.null_count;
      if (c.codec != 0) o << ",\"codec\":" << c.codec << ",\"lz4_device_pages\":" << c.lz4_pages;
      if (c.has_minmax && c.phys == PT_INT64) o << ",\"min\":" << c.min_bits << ",\"max\":" << c.max_bits;
      // Decode through the same directories / tile indexes the kernel uses (small inputs only).
      if (rg.n_rows <= 65536) {
        std::vector<HostRun> vruns, druns;
        if (d.runs) vruns.assign(reinterpret_cast<const HostRun*>(d.runs), reinterpret_cast<const HostRun*>(d.runs) + d.n_runs + 1);
        if (d.def_runs) druns.assign(reinterpret_cast<const HostRun*>(d.def_runs), reinterpret_cast<const HostRun*>(d.def_runs) + d.n_defruns + 1);
        const GlobalDict* gd = nullptr;
        if (d.kind == CK_DICT_STR) gd = &table.dicts.at(name);
        o << ",\"decoded\":[";
        uint32_t vord = 0;
        bool tiles_ok = true;
        for (uint32_t r = 0; r < rg.n_rows; r++) {
          if (r) o << ',';
          if (r % T == 0) {
            auto seed_ok = [&](const Seed& sd, const std::vector<HostRun>& runs, uint32_t first, uint32_t total) {
              if (first >= total) return true;
              if (sd.k >= runs.size() - 1) return false;
              const HostRun& rr = runs[sd.k];
              return rr.start <= first && runs[sd.k + 1].start > first && sd.start == rr.start && sd.end == runs[sd.k + 1].start &&
                     sd.off == rr.off && sd.val == rr.val && sd.meta == rr.meta;
            };
            if (d.kind != CK_PLAIN64) {
              const Seed& sd = d.seeds[r / T];
              if (sd.val0 != vord || !seed_ok(sd, vruns, vord, d.n_values)) tiles_ok = false;
            }
            if (d.has_nulls) {
              const Seed& sd = d.def_seeds[r / T];
              if (sd.val0 != vord || !seed_ok(sd, druns, r, rg.n_rows)) tiles_ok = false;
            }
          }
          bool valid = true;
          if (d.has_nulls) valid = hybrid_value_at(d.def, druns, r) != 0;
          if (!valid) { o << "null"; continue; }
          if (d.kind == CK_PLAIN64) {
            int64_t v;
            std::memcpy(&v, d.values + size_t(vord) * 8, 8);
            if (c.phys == PT_DOUBLE) {
              double f;
              std::memcpy(&f, &v, 8);
              char buf[40];
              snprintf(buf, sizeof buf, "%.17g", f);
              o << buf;
            } else o << v;
          } else {
            bool was_rle = false;
            uint32_t idx = hybrid_value_at(d.values, vruns, vord, &was_rle);
            if (d.kind == CK_DICT_STR) json_escape(o, gd->values[was_rle ? idx : d.lut[idx]]);
            else if (c.phys == PT_DOUBLE) {
              double f;
              std::memcpy(&f, &d.dict64[idx], 8);
              char buf[40];
              snprintf(buf, sizeof buf, "%.17g", f);
              o << buf;
            } else o << d.dict64[idx];
          }
          vord++;
        }
        o << "],\"tile_index_ok\":" << (tiles_ok ? "true" : "false");
        // the row-space directory (sorted-run kernel) must say the same as the two streams it was merged from
        if (d.row_runs) {
          std::vector<HostRun> rr(reinterpret_cast<const HostRun*>(d.row_runs), reinterpret_cast<const HostRun*>(d.row_runs) + d.n_row_runs + 1);
          bool ok = rr.back().start == rg.n_rows;
          uint32_t vo = 0;
          for (uint32_t r = 0; r < rg.n_rows && ok; r++) {
            const uint32_t got = hybrid_value_at(nullptr, rr, r);
            const bool valid = !d.has_nulls || hybrid_value_at(d.def, druns, r) != 0;
            if (!valid) { ok = got == 0xffffffffu; continue; }
            bool was_rle = false;
            uint32_t idx = hybrid_value_at(d.values, vruns, vo++, &was_rle);
            ok = got == (was_rle ? idx : d.lut[idx]);
            if (r % T == 0) {
              const Seed& sd = d.row_seeds[r / T];
              ok = ok && sd.k < rr.size() - 1 && rr[sd.k].start <= r && rr[sd.k + 1].start > r && sd.end == rr[sd.k + 1].start && sd.val == rr[sd.k].val;
            }
          }
          o << ",\"n_row_runs\":" << d.n_row_runs << ",\"row_runs_ok\":" << (ok ? "true" : "false");
        }
      }
      o << '}';
    }
    o << "}}";
  }
  o << "]}";
  return o.str();
}

}  // namespace fgpu
