// See parquet_meta.h.  Thrift compact protocol + Parquet metadata structures, written from the
// public format specification (field ids in comments are parquet.thrift's).
#include "parquet_meta.h"

#include <algorithm>
#include <cstring>
#include <type_traits>

namespace fgpu {
namespace {

struct ThriftError {};

// Minimal Thrift *compact* protocol reader with bounds checks.
class TReader {
 public:
  TReader(const uint8_t* p, const uint8_t* end) : p_(p), end_(end) {}
  const uint8_t* pos() const { return p_; }

  uint8_t byte() {
    if (p_ >= end_) throw ThriftError{};
    return *p_++;
  }
  uint64_t uvarint() {
    uint64_t v = 0;
    int shift = 0;
    for (;;) {
      uint8_t b = byte();
      v |= uint64_t(b & 0x7f) << shift;
      if (!(b & 0x80)) return v;
      shift += 7;
      if (shift > 63) throw ThriftError{};
    }
  }
  int64_t zigzag() {
    uint64_t u = uvarint();
    return int64_t(u >> 1) ^ -int64_t(u & 1);
  }
  std::string binary() {
    uint64_t n = uvarint();
    if (n > uint64_t(end_ - p_)) throw ThriftError{};
    std::string s(reinterpret_cast<const char*>(p_), size_t(n));
    p_ += n;
    return s;
  }
  void skip_bytes(uint64_t n) {
    if (n > uint64_t(end_ - p_)) throw ThriftError{};
    p_ += n;
  }

  // Struct field iteration.  Returns false on STOP.  `type` is the compact wire type.
  bool field(int16_t* last_id, int16_t* id, int* type) {
    uint8_t h = byte();
    if (h == 0) return false;
    int delta = h >> 4;
    *type = h & 0x0f;
    if (delta == 0)
      *id = int16_t(zigzag());
    else
      *id = int16_t(*last_id + delta);
    *last_id = *id;
    return true;
  }
  // List header: element type + count.
  void list(int* etype, uint32_t* n) {
    uint8_t h = byte();
    *etype = h & 0x0f;
    uint32_t sz = h >> 4;
    if (sz == 15) sz = uint32_t(uvarint());
    *n = sz;
  }
  void skip(int type, int depth = 0) {
    if (depth > 32) throw ThriftError{};
    switch (type) {
      case 1: case 2: return;             // bool encoded in the field header
      case 3: byte(); return;             // i8
      case 4: case 5: case 6: uvarint(); return;  // i16/i32/i64 (zigzag varint)
      case 7: skip_bytes(8); return;      // double
      case 8: skip_bytes(uvarint()); return;  // binary
      case 9: case 10: {                  // list / set
        int et; uint32_t n;
        list(&et, &n);
        for (uint32_t i = 0; i < n; i++) {
          if (et == 1 || et == 2) byte();  // bools inside lists take one byte
          else skip(et, depth + 1);
        }
        return;
      }
      case 11: {                          // map
        uint64_t n = uvarint();
        if (n == 0) return;
        uint8_t kv = byte();
        for (uint64_t i = 0; i < n; i++) {
          skip(kv >> 4, depth + 1);
          skip(kv & 0x0f, depth + 1);
        }
        return;
      }
      case 12: {                          // struct
        int16_t last = 0, id; int t;
        while (field(&last, &id, &t)) skip(t, depth + 1);
        return;
      }
      default: throw ThriftError{};
    }
  }

 private:
  const uint8_t* p_;
  const uint8_t* end_;
};

struct RawSchemaElement {
  int32_t type = -1, repetition = 0, num_children = 0, converted = -1;
  bool logical_unsigned = false;
  std::string name;
};

void read_logical_type(TReader& r, RawSchemaElement* e) {
  // union LogicalType { ... 10: IntType INTEGER {1: i8 bitWidth, 2: bool isSigned} ... }
  int16_t last = 0, id; int t;
  while (r.field(&last, &id, &t)) {
    if (id == 10 && t == 12) {
      int16_t l2 = 0, id2; int t2;
      while (r.field(&l2, &id2, &t2)) {
        if (id2 == 2 && (t2 == 1 || t2 == 2)) e->logical_unsigned = (t2 == 2);
        else r.skip(t2);
      }
    } else {
      r.skip(t);
    }
  }
}

RawSchemaElement read_schema_element(TReader& r) {
  RawSchemaElement e;
  int16_t last = 0, id; int t;
  while (r.field(&last, &id, &t)) {
    switch (id) {
      case 1: e.type = int32_t(r.zigzag()); break;          // Type
      case 3: e.repetition = int32_t(r.zigzag()); break;    // FieldRepetitionType
      case 4: e.name = r.binary(); break;
      case 5: e.num_children = int32_t(r.zigzag()); break;
      case 6: e.converted = int32_t(r.zigzag()); break;     // ConvertedType
      case 10: read_logical_type(r, &e); break;
      default: r.skip(t);
    }
  }
  return e;
}

struct RawColumnMeta {
  int32_t type = -1, codec = 0;
  int64_t num_values = 0, total_uncompressed = 0, total_compressed = 0, data_page_offset = -1, dict_page_offset = -1;
  int64_t null_count = -1;
  int64_t bloom_offset = -1;
  int32_t bloom_length = -1;
  std::string stat_min, stat_max;  // raw PLAIN-encoded bounds, empty = not written
  bool stat_deprecated = false;    // the bounds come from the deprecated min / max fields (signed byte order for BYTE_ARRAY)
  std::vector<std::string> path;
};

void read_statistics(TReader& r, RawColumnMeta* m) {
  // Statistics {1: max, 2: min, 3: i64 null_count, 4: distinct_count, 5: max_value, 6: min_value, ...}
  // The deprecated pair (1, 2) is ordered by signed comparison, which is the right order for the
  // INT64 / DOUBLE columns the bounds are used on; the new pair wins when both are present.
  std::string old_min, old_max;
  int16_t last = 0, id; int t;
  while (r.field(&last, &id, &t)) {
    if (id == 3) m->null_count = r.zigzag();
    else if (id == 1 && t == 8) old_max = r.binary();
    else if (id == 2 && t == 8) old_min = r.binary();
    else if (id == 5 && t == 8) m->stat_max = r.binary();
    else if (id == 6 && t == 8) m->stat_min = r.binary();
    else r.skip(t);
  }
  if (m->stat_min.empty() || m->stat_max.empty()) {
    m->stat_min = old_min;
    m->stat_max = old_max;
    m->stat_deprecated = true;
  }
}

RawColumnMeta read_column_meta(TReader& r) {
  RawColumnMeta m;
  int16_t last = 0, id; int t;
  while (r.field(&last, &id, &t)) {
    switch (id) {
      case 1: m.type = int32_t(r.zigzag()); break;
      case 3: {
        int et; uint32_t n;
        r.list(&et, &n);
        for (uint32_t i = 0; i < n; i++) m.path.push_back(r.binary());
        break;
      }
      case 4: m.codec = int32_t(r.zigzag()); break;
      case 5: m.num_values = r.zigzag(); break;
      case 6: m.total_uncompressed = r.zigzag(); break;
      case 7: m.total_compressed = r.zigzag(); break;
      case 9: m.data_page_offset = r.zigzag(); break;
      case 11: m.dict_page_offset = r.zigzag(); break;
      case 12: read_statistics(r, &m); break;
      case 14: m.bloom_offset = r.zigzag(); break;
      case 15: m.bloom_length = int32_t(r.zigzag()); break;
      default: r.skip(t);
    }
  }
  return m;
}

// BloomFilterHeader {1: i32 numBytes, 2: BloomFilterAlgorithm {1: BLOCK}, 3: BloomFilterHash {1: XXHASH},
// 4: BloomFilterCompression {1: UNCOMPRESSED}} followed by the bitset.  Anything else: the filter is ignored.
void read_bloom(const uint8_t* file, uint64_t len, int64_t offset, ChunkMeta* out) {
  if (offset < 0 || uint64_t(offset) >= len) return;
  try {
    TReader r(file + offset, file + len);
    int32_t num_bytes = -1;
    bool ok = true;
    int16_t last = 0, id; int t;
    auto union_is_1 = [&](TReader& rr) {  // a union with exactly field 1 set (an empty struct)
      bool one = false;
      int16_t l2 = 0, id2; int t2;
      while (rr.field(&l2, &id2, &t2)) {
        if (id2 == 1) one = true;
        else one = false;
        rr.skip(t2);
      }
      return one;
    };
    while (r.field(&last, &id, &t)) {
      if (id == 1) num_bytes = int32_t(r.zigzag());
      else if ((id == 2 || id == 3 || id == 4) && t == 12) ok = union_is_1(r) && ok;
      else r.skip(t);
    }
    if (!ok || num_bytes < 32 || num_bytes % 32 != 0) return;
    if (uint64_t(r.pos() - file) + uint64_t(num_bytes) > len) return;
    out->bloom = r.pos();
    out->bloom_bytes = uint32_t(num_bytes);
  } catch (ThriftError&) {
  }
}

struct RawPageHeader {
  int32_t type = -1, uncompressed = 0, compressed = 0;
  // data page v1 / v2 / dictionary
  int32_t num_values = 0, encoding = 0, def_encoding = ENC_RLE, rep_encoding = ENC_RLE;
  int32_t num_nulls = -1, num_rows = 0, def_len = 0, rep_len = 0;
  bool v2_compressed = true;
};

void read_data_page_header(TReader& r, RawPageHeader* h) {
  int16_t last = 0, id; int t;
  while (r.field(&last, &id, &t)) {
    switch (id) {
      case 1: h->num_values = int32_t(r.zigzag()); break;
      case 2: h->encoding = int32_t(r.zigzag()); break;
      case 3: h->def_encoding = int32_t(r.zigzag()); break;
      case 4: h->rep_encoding = int32_t(r.zigzag()); break;
      default: r.skip(t);
    }
  }
}
void read_dict_page_header(TReader& r, RawPageHeader* h) {
  int16_t last = 0, id; int t;
  while (r.field(&last, &id, &t)) {
    switch (id) {
      case 1: h->num_values = int32_t(r.zigzag()); break;
      case 2: h->encoding = int32_t(r.zigzag()); break;
      default: r.skip(t);
    }
  }
}
void read_data_page_header_v2(TReader& r, RawPageHeader* h) {
  int16_t last = 0, id; int t;
  while (r.field(&last, &id, &t)) {
    switch (id) {
      case 1: h->num_values = int32_t(r.zigzag()); break;
      case 2: h->num_nulls = int32_t(r.zigzag()); break;
      case 3: h->num_rows = int32_t(r.zigzag()); break;
      case 4: h->encoding = int32_t(r.zigzag()); break;
      case 5: h->def_len = int32_t(r.zigzag()); break;
      case 6: h->rep_len = int32_t(r.zigzag()); break;
      case 7: h->v2_compressed = (t == 1); break;
      default: r.skip(t);
    }
  }
}

RawPageHeader read_page_header(TReader& r) {
  RawPageHeader h;
  int16_t last = 0, id; int t;
  while (r.field(&last, &id, &t)) {
    switch (id) {
      case 1: h.type = int32_t(r.zigzag()); break;
      case 2: h.uncompressed = int32_t(r.zigzag()); break;
      case 3: h.compressed = int32_t(r.zigzag()); break;
      case 5: read_data_page_header(r, &h); break;
      case 7: read_dict_page_header(r, &h); break;
      case 8: read_data_page_header_v2(r, &h); break;
      default: r.skip(t);
    }
  }
  return h;
}

// Footer facts of one column chunk (no page is touched).
void init_chunk(const RawColumnMeta& cm, const SchemaLeaf& leaf, ChunkMeta* out) {
  out->data_page_offset = cm.data_page_offset;
  out->dict_page_offset = cm.dict_page_offset;
  out->codec = cm.codec;
  out->num_values = cm.num_values;
  out->total_compressed_size = cm.total_compressed;
  out->total_uncompressed_size = cm.total_uncompressed;
  out->null_count = cm.null_count;
  if ((leaf.phys == PT_INT64 || leaf.phys == PT_DOUBLE) && cm.stat_min.size() == 8 && cm.stat_max.size() == 8) {
    out->has_minmax = true;
    std::memcpy(&out->min_bits, cm.stat_min.data(), 8);
    std::memcpy(&out->max_bits, cm.stat_max.data(), 8);
  }
  // string bounds: min_value / max_value only (legacy writers order the deprecated pair by signed bytes)
  if (leaf.phys == PT_BYTE_ARRAY && !cm.stat_deprecated && !cm.stat_min.empty() && !cm.stat_max.empty()) {
    out->has_minmax_str = true;
    out->min_str = cm.stat_min;
    out->max_str = cm.stat_max;
  }
  if (cm.codec != 0 && cm.codec != kCodecLz4Raw) {
    out->error = "compressed column chunk (codec " + std::to_string(cm.codec) + ") is not supported";
    return;
  }
  if (leaf.max_rep > 0) {
    out->error = "repeated (nested) columns are not supported";
    return;
  }
}

}  // namespace

namespace {

// LZ4_RAW chunks: the device inflates the values of PLAIN INT64 / DOUBLE pages whose block holds nothing but values
// (data page v2 of any column, data page v1 of a REQUIRED column); the host inflates every other page.
bool plain_numeric(const SchemaLeaf& leaf, const RawPageHeader& h) {
  return h.encoding == ENC_PLAIN && (leaf.phys == PT_INT64 || leaf.phys == PT_DOUBLE);
}
bool device_inflates(const SchemaLeaf& leaf, const RawPageHeader& h) {
  if (!plain_numeric(leaf, h)) return false;
  return h.type == PG_DATA_V2 ? h.v2_compressed : (h.type == PG_DATA && leaf.max_def == 0);
}

// Bytes a page of an LZ4_RAW chunk adds to ChunkMeta::inflated (its values region, or all of a v1 page; the levels of a
// v2 page stay in the file).  Nonsense sizes count 0: the walk refuses the page before it inflates anything.
uint64_t host_inflated_bytes(const SchemaLeaf& leaf, const RawPageHeader& h) {
  if (h.type != PG_DICTIONARY && h.type != PG_DATA && h.type != PG_DATA_V2) return 0;
  if (h.type == PG_DATA_V2 ? plain_numeric(leaf, h) : (h.type == PG_DATA && device_inflates(leaf, h))) return 0;
  const int64_t raw = h.type == PG_DATA_V2 ? int64_t(h.uncompressed) - h.def_len - h.rep_len : int64_t(h.uncompressed);
  return raw > 0 ? uint64_t(raw) : 0;
}

}  // namespace

void walk_chunk_pages(const uint8_t* file, uint64_t len, const SchemaLeaf& leaf, int64_t rg_rows, ChunkMeta* out) {
  if (out->pages_walked) return;
  out->pages_walked = true;
  if (!out->error.empty()) return;
  struct { int64_t data_page_offset, dict_page_offset, total_compressed, num_values; } cm{out->data_page_offset, out->dict_page_offset,
                                                                                          out->total_compressed_size, out->num_values};
  int64_t start = cm.data_page_offset;
  if (cm.dict_page_offset > 0 && cm.dict_page_offset < start) start = cm.dict_page_offset;
  if (start < 4 || uint64_t(start) >= len) {
    out->error = "column chunk offset out of range";
    return;
  }
  const uint8_t* p = file + start;
  const uint8_t* end = file + len;
  // total_compressed_size bounds the chunk (headers included).
  if (cm.total_compressed > 0 && uint64_t(start) + uint64_t(cm.total_compressed) <= len)
    end = p + cm.total_compressed;
  const uint8_t* const first = p;
  const bool lz4 = out->codec == kCodecLz4Raw;
  if (lz4) {
    // sizing pass: the host-inflated bytes of every page go into one buffer, allocated once (pointers into it stay valid);
    // the walk below reports whatever stops this pass
    uint64_t bytes = 0;
    int64_t seen = 0;
    try {
      while (seen < cm.num_values && p < end) {
        TReader r(p, end);
        const RawPageHeader h = read_page_header(r);
        if (h.compressed < 0 || uint64_t(h.compressed) > uint64_t(end - r.pos())) break;
        if (h.uncompressed >= 0 && uint64_t(h.uncompressed) <= 256 * uint64_t(h.compressed)) bytes += host_inflated_bytes(leaf, h);
        if (h.type == PG_DATA || h.type == PG_DATA_V2) seen += h.num_values;
        p = r.pos() + h.compressed;
      }
    } catch (ThriftError&) {
    }
    out->inflated.assign(size_t(bytes) + 8, 0);  // (8 pad bytes: hybrid streams are read in 5-byte windows)
    p = first;
  }
  uint64_t at = 0;  // fill of `inflated`
  // the `raw` bytes that `n` stored bytes at `src` stand for, inflated into `inflated` (LZ4_RAW) or copied there
  // (`compressed` false: a v2 values region stored as is); false with `error` set when the block is refused
  auto inflate = [&](const uint8_t* src, uint32_t n, int64_t raw, bool compressed, const uint8_t** dst) {
    if (raw < 0 || (compressed && n > 0 && uint64_t(raw) > 256 * uint64_t(n))) {
      out->error = "LZ4_RAW page size out of range";
      return false;
    }
    if (at + uint64_t(raw) > out->inflated.size() - 8) {
      out->error = "LZ4_RAW page sizes changed between two reads";
      return false;
    }
    uint8_t* q = out->inflated.data() + at;
    if (!compressed) {
      if (uint64_t(raw) != n) { out->error = "uncompressed v2 values region differs from its page's size"; return false; }
      if (n) std::memcpy(q, src, n);
    } else if (n != 0 || raw != 0) {  // (an empty region may be stored as 0 bytes)
      std::string e;
      if (!parse_lz4_raw(src, n, uint64_t(raw), &e)) { out->error = e; return false; }
      unpack_lz4_raw(src, n, q, uint64_t(raw));
    }
    at += uint64_t(raw);
    *dst = q;
    return true;
  };
  // a device-inflated values region: validated only (parse step), left in the file
  auto validate = [&](PageInfo* pg, int64_t raw) {
    if (raw < 0 || (pg->values_len > 0 && uint64_t(raw) > 256 * uint64_t(pg->values_len))) {
      out->error = "LZ4_RAW page size out of range";
      return false;
    }
    if (pg->values_len == 0 && raw == 0) return true;
    std::string e;
    if (!parse_lz4_raw(pg->values, pg->values_len, uint64_t(raw), &e)) { out->error = e; return false; }
    if (raw == 0) pg->values_len = 0;  // (the block 0x00: no values)
    pg->lz4_len = uint32_t(raw);
    return true;
  };
  int64_t values_seen = 0;
  try {
    while (values_seen < cm.num_values && p < end) {
      TReader r(p, end);
      RawPageHeader h = read_page_header(r);
      const uint8_t* payload = r.pos();
      if (h.compressed < 0 || uint64_t(h.compressed) > uint64_t(end - payload)) {
        out->error = "page payload overruns chunk";
        return;
      }
      if (h.type == PG_DICTIONARY) {
        if (h.encoding != ENC_PLAIN && h.encoding != ENC_PLAIN_DICTIONARY) {
          out->error = "dictionary page with non-PLAIN encoding";
          return;
        }
        out->dict = payload;
        out->dict_len = uint32_t(h.compressed);
        if (lz4) {
          if (!inflate(payload, uint32_t(h.compressed), h.uncompressed, true, &out->dict)) return;
          out->dict_len = uint32_t(h.uncompressed);
        }
        out->dict_num_values = uint32_t(h.num_values);
      } else if (h.type == PG_DATA) {
        PageInfo pg;
        pg.type = PG_DATA;
        pg.encoding = h.encoding;
        pg.num_values = uint32_t(h.num_values);
        const uint8_t* q = payload;
        const uint8_t* pend = payload + h.compressed;
        if (lz4 && !device_inflates(leaf, h)) {  // levels and values are one block
          if (!inflate(payload, uint32_t(h.compressed), h.uncompressed, true, &q)) return;
          pend = q + h.uncompressed;
        }
        if (leaf.max_def > 0) {
          if (h.def_encoding != ENC_RLE) {
            out->error = "v1 page with non-RLE definition levels";
            return;
          }
          if (pend - q < 4) { out->error = "truncated definition levels"; return; }
          uint32_t dl;
          std::memcpy(&dl, q, 4);
          q += 4;
          if (dl > uint64_t(pend - q)) { out->error = "definition levels overrun page"; return; }
          pg.def = q;
          pg.def_len = dl;
          q += dl;
        }
        pg.values = q;
        pg.values_len = uint32_t(pend - q);
        if (lz4 && device_inflates(leaf, h) && !validate(&pg, h.uncompressed)) return;
        values_seen += h.num_values;
        out->pages.push_back(pg);
      } else if (h.type == PG_DATA_V2) {
        PageInfo pg;
        pg.type = PG_DATA_V2;
        pg.encoding = h.encoding;
        pg.num_values = uint32_t(h.num_values);
        pg.num_nulls = h.num_nulls;
        if (h.rep_len != 0) { out->error = "repetition levels present"; return; }
        if (h.def_len < 0 || h.def_len > h.compressed) { out->error = "bad v2 level length"; return; }
        pg.def = payload;
        pg.def_len = uint32_t(h.def_len);
        pg.values = payload + h.def_len;
        pg.values_len = uint32_t(h.compressed - h.def_len);
        if (lz4) {  // the levels are stored as they are, the values region is one block unless is_compressed says otherwise
          const int64_t raw = int64_t(h.uncompressed) - h.def_len;
          if (device_inflates(leaf, h)) {
            if (!validate(&pg, raw)) return;
          } else if (!plain_numeric(leaf, h)) {
            if (!inflate(pg.values, pg.values_len, raw, h.v2_compressed, &pg.values)) return;
            pg.values_len = uint32_t(raw);
          } else if (raw != int64_t(pg.values_len)) {  // PLAIN numeric values stored as they are: read from the file
            out->error = "uncompressed v2 values region differs from its page's size";
            return;
          }
        }
        values_seen += h.num_values;
        out->pages.push_back(pg);
      }  // index pages and unknown page types are skipped
      p = payload + h.compressed;
    }
  } catch (ThriftError&) {
    out->error = "malformed page header";
    return;
  }
  if (values_seen != cm.num_values) {
    out->error = "page walk found " + std::to_string(values_seen) + " values, footer says " +
                 std::to_string(cm.num_values);
    return;
  }
  if (cm.num_values != rg_rows) {
    out->error = "flat column with num_values != row group rows";
    return;
  }
}

bool parse_parquet(const uint8_t* file, uint64_t len, ParsedFile* out, std::string* err, bool walk_pages) {
  *out = ParsedFile{};
  if (len < 12 || std::memcmp(file, "PAR1", 4) != 0 || std::memcmp(file + len - 4, "PAR1", 4) != 0) {
    *err = "not a Parquet file (missing PAR1 magic)";
    return false;
  }
  uint32_t flen;
  std::memcpy(&flen, file + len - 8, 4);
  if (uint64_t(flen) + 12 > len) {
    *err = "footer length out of range";
    return false;
  }
  const uint8_t* fstart = file + len - 8 - flen;
  std::vector<RawSchemaElement> schema;
  struct RawRG { int64_t num_rows = 0; std::vector<RawColumnMeta> cols; };
  std::vector<RawRG> rgs;
  try {
    TReader r(fstart, fstart + flen);
    int16_t last = 0, id; int t;
    while (r.field(&last, &id, &t)) {
      switch (id) {
        case 2: {  // schema
          int et; uint32_t n;
          r.list(&et, &n);
          for (uint32_t i = 0; i < n; i++) schema.push_back(read_schema_element(r));
          break;
        }
        case 3: out->num_rows = r.zigzag(); break;
        case 4: {  // row_groups
          int et; uint32_t n;
          r.list(&et, &n);
          for (uint32_t i = 0; i < n; i++) {
            RawRG rg;
            int16_t l2 = 0, id2; int t2;
            while (r.field(&l2, &id2, &t2)) {
              if (id2 == 1) {  // columns
                int et2; uint32_t n2;
                r.list(&et2, &n2);
                for (uint32_t j = 0; j < n2; j++) {
                  RawColumnMeta cm;
                  int16_t l3 = 0, id3; int t3;
                  while (r.field(&l3, &id3, &t3)) {  // ColumnChunk
                    if (id3 == 3) cm = read_column_meta(r);
                    else r.skip(t3);
                  }
                  rg.cols.push_back(std::move(cm));
                }
              } else if (id2 == 3) {
                rg.num_rows = r.zigzag();
              } else {
                r.skip(t2);
              }
            }
            rgs.push_back(std::move(rg));
          }
          break;
        }
        case 5: {  // key_value_metadata
          int et; uint32_t n;
          r.list(&et, &n);
          for (uint32_t i = 0; i < n; i++) {
            std::string k, v;
            int16_t l2 = 0, id2; int t2;
            while (r.field(&l2, &id2, &t2)) {
              if (id2 == 1) k = r.binary();
              else if (id2 == 2) v = r.binary();
              else r.skip(t2);
            }
            out->kv.emplace_back(std::move(k), std::move(v));
          }
          break;
        }
        case 6: out->created_by = r.binary(); break;
        default: r.skip(t);
      }
    }
  } catch (ThriftError&) {
    *err = "malformed Parquet footer";
    return false;
  }
  if (schema.empty()) {
    *err = "empty schema";
    return false;
  }
  // Flatten the schema tree (depth first) into leaves with dotted paths and level maxima.
  {
    struct Frame { int remaining; std::string prefix; int def, rep; };
    std::vector<Frame> stack;
    stack.push_back({schema[0].num_children, "", 0, 0});
    for (size_t i = 1; i < schema.size(); i++) {
      while (!stack.empty() && stack.back().remaining == 0) stack.pop_back();
      if (stack.empty()) { *err = "schema tree malformed"; return false; }
      Frame& f = stack.back();
      f.remaining--;
      const RawSchemaElement& e = schema[i];
      int def = f.def + (e.repetition != 0 ? 1 : 0);
      int rep = f.rep + (e.repetition == 2 ? 1 : 0);
      std::string path = f.prefix.empty() ? e.name : f.prefix + "." + e.name;
      if (e.num_children > 0) {
        stack.push_back({e.num_children, path, def, rep});
      } else {
        SchemaLeaf leaf;
        leaf.name = path;
        leaf.phys = e.type;
        leaf.max_def = def;
        leaf.max_rep = rep;
        leaf.is_unsigned = e.logical_unsigned || e.converted == 14 /*UINT_64*/;
        out->leaves.push_back(std::move(leaf));
      }
    }
  }
  for (auto& rg : rgs) {
    if (rg.cols.size() != out->leaves.size()) {
      *err = "row group column count does not match schema leaves";
      return false;
    }
    RowGroupMeta m;
    m.num_rows = rg.num_rows;
    m.chunks.resize(rg.cols.size());
    for (size_t c = 0; c < rg.cols.size(); c++) {
      m.chunks[c].leaf = int32_t(c);
      init_chunk(rg.cols[c], out->leaves[c], &m.chunks[c]);
      if (rg.cols[c].bloom_offset >= 0) read_bloom(file, len, rg.cols[c].bloom_offset, &m.chunks[c]);
      if (walk_pages) walk_chunk_pages(file, len, out->leaves[c], rg.num_rows, &m.chunks[c]);
    }
    out->row_groups.push_back(std::move(m));
  }
  return true;
}

bool walk_hybrid(const uint8_t* data, uint32_t len, int w, uint32_t count, uint32_t start0,
                 uint32_t off0, std::vector<HostRun>* runs, std::string* err) {
  const uint8_t* p = data;
  const uint8_t* end = data + len;
  uint32_t produced = 0;
  const uint32_t vbytes = uint32_t((w + 7) / 8);
  constexpr uint32_t kShortLiteral = 64;
  // appends a run-length entry, merging with a preceding one of the same value (also the last run of
  // the previous page of the chunk: `runs` is per column chunk and its runs are contiguous, the
  // previous run ends where this one starts)
  auto push_rle = [&](uint32_t start, uint32_t v) {
    if (!runs->empty() && (runs->back().meta & 1u) == 0 && runs->back().val == v) return;
    HostRun r;
    r.start = start;
    r.off = 0;
    r.val = v;
    r.meta = 0u | (uint32_t(w) << 8);
    runs->push_back(r);
  };
  while (produced < count) {
    // ULEB128 run header
    uint64_t h = 0;
    int shift = 0;
    for (;;) {
      if (p >= end) { *err = "hybrid stream truncated (header)"; return false; }
      uint8_t b = *p++;
      h |= uint64_t(b & 0x7f) << shift;
      if (!(b & 0x80)) break;
      shift += 7;
      if (shift > 35) { *err = "hybrid run header too long"; return false; }
    }
    if (h & 1) {  // bit-packed: (h >> 1) groups of 8 values
      uint64_t groups = h >> 1;
      uint64_t nvals = groups * 8;
      uint64_t nbytes = groups * uint64_t(w);
      // The last group of a stream may be cut short by writers that trim padding.
      uint64_t avail = uint64_t(end - p);
      if (nbytes > avail) {
        uint64_t need_vals = count - produced;
        uint64_t need_bytes = (need_vals * uint64_t(w) + 7) / 8;
        if (need_bytes > avail) { *err = "hybrid stream truncated (bit-packed run)"; return false; }
        nbytes = avail;
      }
      uint32_t take = uint32_t(nvals < uint64_t(count - produced) ? nvals : uint64_t(count - produced));
      if (take > 0 && w == 0) {
        // a width-0 literal (one-entry dictionary) is a run of index 0 of any length: recorded as one, it keeps
        // such a column run-length only
        push_rle(start0 + produced, 0);
      } else if (take > 0 && take <= kShortLiteral) {
        // Writers close a repeated run on a multiple of 8 values and spill the boundary into one or two
        // literal groups ("aaaaabbb").  Such short literal runs are unpacked here into run-length
        // entries, so the directory of a sorted column holds no bit-packed run at all and the scan
        // kernel's run cursor never has to unpack bits at a group boundary.
        for (uint32_t i = 0; i < take; i++) {
          uint64_t bit = uint64_t(i) * uint64_t(w);
          uint64_t word = 0;
          const uint8_t* q = p + (bit >> 3);
          if (end - q >= 8) std::memcpy(&word, q, 8);
          else for (int b = 0; b < 8 && q + b < end; b++) word |= uint64_t(q[b]) << (8 * b);
          uint32_t v = w == 0 ? 0u : uint32_t((word >> (bit & 7)) & ((w >= 32 ? 0xffffffffull : ((1ull << w) - 1))));
          push_rle(start0 + produced + i, v);
        }
      } else if (take > 0) {
        HostRun r;
        r.start = start0 + produced;
        r.off = off0 + uint32_t(p - data);
        r.val = 0;
        r.meta = 1u | (uint32_t(w) << 8);
        runs->push_back(r);
      }
      produced += take;
      p += nbytes;
    } else {  // RLE: (h >> 1) copies of one value in ceil(w/8) bytes
      uint64_t n = h >> 1;
      if (uint64_t(end - p) < vbytes) { *err = "hybrid stream truncated (RLE value)"; return false; }
      uint32_t v = 0;
      for (uint32_t i = 0; i < vbytes; i++) v |= uint32_t(p[i]) << (8 * i);
      p += vbytes;
      uint32_t take = uint32_t(n < uint64_t(count - produced) ? n : uint64_t(count - produced));
      if (take > 0) push_rle(start0 + produced, v);
      produced += take;
      if (n == 0) { *err = "zero-length RLE run"; return false; }
    }
  }
  return true;
}

uint32_t hybrid_value_at(const uint8_t* stream, const std::vector<HostRun>& runs, uint32_t ordinal, bool* was_rle) {
  // binary search the last run with start <= ordinal
  size_t lo = 0, hi = runs.size();
  while (hi - lo > 1) {
    size_t mid = (lo + hi) / 2;
    if (runs[mid].start <= ordinal) lo = mid; else hi = mid;
  }
  const HostRun& r = runs[lo];
  if (was_rle) *was_rle = (r.meta & 1u) == 0;
  if ((r.meta & 1u) == 0) return r.val;
  uint32_t w = (r.meta >> 8) & 0xff;
  if (w == 0) return 0;
  uint64_t bit = uint64_t(ordinal - r.start) * w;
  const uint8_t* p = stream + r.off + (bit >> 3);
  uint64_t window = 0;
  for (int i = 0; i < 5; i++) window |= uint64_t(p[i]) << (8 * i);  // callers pad streams by 8 bytes
  return uint32_t((window >> (bit & 7)) & ((w == 32) ? 0xffffffffull : ((1ull << w) - 1)));
}

// ---- DELTA_BINARY_PACKED -------------------------------------------------------------------------------------
namespace {
bool read_uleb(const uint8_t*& p, const uint8_t* end, uint64_t* v) {
  uint64_t x = 0;
  for (int shift = 0; shift < 70; shift += 7) {
    if (p >= end) return false;
    const uint8_t b = *p++;
    if (shift < 64) x |= uint64_t(b & 0x7f) << shift;
    if ((b & 0x80) == 0) {
      *v = x;
      return true;
    }
  }
  return false;
}
}  // namespace

template <typename T>
bool parse_delta_binary_packed(const uint8_t* data, uint64_t len, uint32_t count, DbpStream* out, std::string* err) {
  using U = typename std::make_unsigned<T>::type;
  constexpr uint32_t kBits = 8 * sizeof(T);
  const uint8_t* p = data;
  const uint8_t* const end = data + len;
  const std::string overrun = "DELTA_BINARY_PACKED stream overruns its page";
  uint64_t block = 0, n_mb = 0, total = 0, first = 0;
  if (!read_uleb(p, end, &block) || !read_uleb(p, end, &n_mb) || !read_uleb(p, end, &total) || !read_uleb(p, end, &first)) {
    *err = overrun;
    return false;
  }
  if (block == 0 || block % 128 != 0) { *err = "DELTA_BINARY_PACKED block size is not a multiple of 128"; return false; }
  if (n_mb == 0 || block % n_mb != 0 || (block / n_mb) % 32 != 0) { *err = "DELTA_BINARY_PACKED miniblock size is not a multiple of 32"; return false; }
  if (total != count) { *err = "DELTA_BINARY_PACKED value count differs from the page's values"; return false; }
  const uint64_t per_mb = block / n_mb;
  if (per_mb > (uint64_t(1) << 40) && count > 1) { *err = overrun; return false; }  // (a miniblock larger than any page)
  out->first = uint64_t(U((first >> 1) ^ (~(first & 1) + 1)));  // zigzag, wrapped to the value width
  out->count = count;
  out->per_mb = per_mb;
  out->mbs.clear();
  uint64_t produced = count > 0 ? 1 : 0;
  while (produced < count) {
    uint64_t zmin = 0;
    if (!read_uleb(p, end, &zmin)) { *err = overrun; return false; }
    const uint64_t min_delta = uint64_t(U((zmin >> 1) ^ (~(zmin & 1) + 1)));
    if (uint64_t(end - p) < n_mb) { *err = overrun; return false; }
    const uint8_t* widths = p;
    p += n_mb;
    for (uint64_t m = 0; m < n_mb && produced < count; m++) {
      const uint32_t w = widths[m];
      if (w > kBits) { *err = "DELTA_BINARY_PACKED miniblock bit width > " + std::to_string(kBits); return false; }
      const uint64_t bytes = per_mb * w / 8;  // a miniblock holding values is written whole (padding included)
      if (uint64_t(end - p) < bytes) { *err = overrun; return false; }
      const uint64_t take = std::min<uint64_t>(per_mb, count - produced);
      out->mbs.push_back(DbpMiniblock{uint64_t(p - data), min_delta, uint32_t(produced), uint32_t(take), w});
      produced += take;
      p += bytes;
    }
  }
  out->used = uint64_t(p - data);
  return true;
}

template <typename T>
void unpack_delta_binary_packed(const uint8_t* data, T first, const DbpMiniblock* mbs, size_t n_mbs, uint32_t ord0, T* out) {
  using U = typename std::make_unsigned<T>::type;
  U v = U(first);
  out[0] = first;
  for (size_t m = 0; m < n_mbs; m++) {
    const DbpMiniblock& mb = mbs[m];
    const uint8_t* p = data + mb.off;
    const uint32_t w = mb.width;
    const uint64_t bytes = (uint64_t(mb.count) * w + 7) / 8;  // (the bytes its values need: the padding is not read)
    T* dst = out + (mb.first - ord0);
    for (uint64_t i = 0; i < mb.count; i++) {
      uint64_t d = 0;
      if (w) {  // LSB first; a 64-bit value at an odd bit position spans 9 bytes
        const uint64_t b0 = (i * w) >> 3, avail = bytes - b0;
        const unsigned sh = unsigned((i * w) & 7);
        uint64_t window = 0;
        for (uint64_t k = 0; k < std::min<uint64_t>(8, avail); k++) window |= uint64_t(p[b0 + k]) << (8 * k);
        d = window >> sh;
        if (sh && avail > 8) d |= uint64_t(p[b0 + 8]) << (64 - sh);
        if (w < 64) d &= (uint64_t(1) << w) - 1;
      }
      v = U(v + U(mb.min_delta) + U(d));
      dst[i] = T(v);
    }
  }
}

template <typename T>
bool decode_delta_binary_packed(const uint8_t* data, uint64_t len, uint32_t count, std::vector<T>* out, uint64_t* used, std::string* err) {
  DbpStream s;
  if (!parse_delta_binary_packed<T>(data, len, count, &s, err)) return false;
  out->assign(count, T(0));
  if (count > 0) unpack_delta_binary_packed<T>(data, T(s.first), s.mbs.data(), s.mbs.size(), 0, out->data());
  *used = s.used;
  return true;
}

template bool parse_delta_binary_packed<int64_t>(const uint8_t*, uint64_t, uint32_t, DbpStream*, std::string*);
template void unpack_delta_binary_packed<int64_t>(const uint8_t*, int64_t, const DbpMiniblock*, size_t, uint32_t, int64_t*);
template bool decode_delta_binary_packed<int32_t>(const uint8_t*, uint64_t, uint32_t, std::vector<int32_t>*, uint64_t*, std::string*);

// ---- LZ4_RAW blocks ---------------------------------------------------------------------------------------------
// A block is a chain of sequences: a token (high nibble: literal length, low nibble: match length - 4, 15 in either
// extended by bytes up to and including the first that is not 255), the literals, then for every sequence but the last a
// 2-byte little-endian offset and the match length extension.  liblz4's decoder adds the end-of-block rules checked here.

bool parse_lz4_raw(const uint8_t* src, uint64_t len, uint64_t out_len, std::string* err) {
  auto bad = [&](const char* m) {
    *err = std::string("LZ4_RAW block: ") + m;
    return false;
  };
  if (len == 0) return bad("empty (a block holds at least one token)");
  if (out_len == 0) {  // (liblz4 takes the one block 0x00 for an empty output)
    if (src[0] >> 4) return bad("output longer than the header says");
    if (src[0] != 0) return bad("the empty output's block is not 0x00");
    return len == 1 ? true : bad("bytes behind the last sequence");
  }
  uint64_t ip = 0, op = 0;
  for (;;) {
    if (ip >= len) return bad("block ends without a sequence without a match");
    const uint32_t token = src[ip++];
    uint64_t lit = token >> 4;
    if (lit == 15) {  // the extension stops at the block's last 15 bytes (they hold at least its literals)
      if (len < 15 || ip >= len - 15) return bad("literal length extension runs past the block");
      for (;;) {
        const uint8_t b = src[ip++];
        lit += b;
        if (ip > len - 15) return bad("literal length extension runs past the block");
        if (b != 255) break;
      }
    }
    if (lit > len - ip) return bad("literal run runs past the block");
    if (lit > out_len - op) return bad("output longer than the header says");
    // the last sequence: its literals reach into the output's last 12 bytes or the block's last 8
    if (op + lit + 12 > out_len || ip + lit + 8 > len) {
      if (ip + lit != len)
        return bad(op + lit == out_len ? "bytes behind the last sequence"
                                       : "a match starts in the last 12 bytes of the output or the last 8 of the block");
      if (op + lit != out_len) return bad("output shorter than the header says");
      return true;
    }
    ip += lit;
    op += lit;
    const uint64_t offset = uint64_t(src[ip]) | (uint64_t(src[ip + 1]) << 8);
    ip += 2;
    if (offset == 0) return bad("match offset 0");
    if (offset > op) return bad("match offset reaches before the start of the output");
    uint64_t ml = token & 15u;
    if (ml == 15) {  // the extension stops at the block's last 4 bytes
      for (;;) {
        const uint8_t b = src[ip++];
        ml += b;
        if (ip > len - 4) return bad("match length extension runs past the block");
        if (b != 255) break;
      }
    }
    ml += 4;
    if (ml > out_len - op) return bad("output longer than the header says");
    if (op + ml + 5 > out_len) return bad("a match ends in the last 5 bytes of the output");
    op += ml;
  }
}

void unpack_lz4_raw(const uint8_t* src, uint64_t len, uint8_t* dst, uint64_t cap) {
  uint64_t ip = 0, op = 0;
  while (ip < len && op < cap) {
    const uint32_t token = src[ip++];
    uint64_t lit = token >> 4;
    if (lit == 15)
      for (uint8_t b = 255; b == 255 && ip < len;) lit += (b = src[ip++]);
    const uint64_t take = std::min(lit, std::min(len - ip, cap - op));
    std::memcpy(dst + op, src + ip, size_t(take));
    ip += lit;
    op += take;
    if (ip + 2 > len || op >= cap) break;
    const uint64_t offset = uint64_t(src[ip]) | (uint64_t(src[ip + 1]) << 8);
    ip += 2;
    uint64_t ml = token & 15u;
    if (ml == 15)
      for (uint8_t b = 255; b == 255 && ip < len;) ml += (b = src[ip++]);
    ml += 4;
    if (offset == 0 || offset > op) break;
    for (const uint64_t e = std::min(cap, op + ml); op < e; op++) dst[op] = dst[op - offset];  // (overlapping: byte by byte)
  }
}

// ---- bloom filters ---------------------------------------------------------------------------------------------
namespace {
constexpr uint64_t kP1 = 11400714785074694791ull, kP2 = 14029467366897019727ull, kP3 = 1609587929392839161ull,
                   kP4 = 9650029242287828579ull, kP5 = 2870177450012600261ull;
inline uint64_t rotl64(uint64_t x, int r) { return (x << r) | (x >> (64 - r)); }
inline uint64_t rd64(const uint8_t* p) { uint64_t v; std::memcpy(&v, p, 8); return v; }
inline uint32_t rd32(const uint8_t* p) { uint32_t v; std::memcpy(&v, p, 4); return v; }
inline uint64_t xx_round(uint64_t acc, uint64_t in) { return rotl64(acc + in * kP2, 31) * kP1; }
inline uint64_t xx_merge(uint64_t acc, uint64_t v) { return (acc ^ xx_round(0, v)) * kP1 + kP4; }
constexpr uint32_t kSalt[8] = {0x47b6137bu, 0x44974d91u, 0x8824ad5bu, 0xa2b7289du, 0x705495c7u, 0x2df1424bu, 0x9efc4947u, 0x5c6bfb31u};
}  // namespace

uint64_t xxhash64(const uint8_t* p, size_t len, uint64_t seed) {
  const uint8_t* const end = p + len;
  uint64_t h;
  if (len >= 32) {
    uint64_t v1 = seed + kP1 + kP2, v2 = seed + kP2, v3 = seed, v4 = seed - kP1;
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
    h = seed + kP5;
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

bool sbbf_check(const uint8_t* bitset, uint32_t bytes, uint64_t hash) {
  const uint64_t n_blocks = bytes / 32;
  if (n_blocks == 0) return true;
  const uint64_t block = ((hash >> 32) * n_blocks) >> 32;
  const uint32_t key = uint32_t(hash);
  const uint8_t* b = bitset + block * 32;
  for (int i = 0; i < 8; i++) {
    const uint32_t bit = 1u << ((key * kSalt[i]) >> 27);
    if ((rd32(b + 4 * i) & bit) == 0) return false;
  }
  return true;
}

void sbbf_insert(uint8_t* bitset, uint32_t bytes, uint64_t hash) {
  const uint64_t n_blocks = bytes / 32;
  if (n_blocks == 0) return;
  const uint64_t block = ((hash >> 32) * n_blocks) >> 32;
  const uint32_t key = uint32_t(hash);
  uint8_t* b = bitset + block * 32;
  for (int i = 0; i < 8; i++) {
    uint32_t w = rd32(b + 4 * i) | (1u << ((key * kSalt[i]) >> 27));
    std::memcpy(b + 4 * i, &w, 4);
  }
}

}  // namespace fgpu
