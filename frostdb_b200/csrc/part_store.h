// Device-resident part registry: what Table.Iterator / LSM.Scan enumerate in the reference
// (table.go:740-868, index/lsm.go:401-454) lives here as a list of parts whose column chunks are
// already laid out in HBM for the scan kernel.
#pragma once
#include <cstdint>
#include <cstring>
#include <map>
#include <memory>
#include <string>
#include <string_view>
#include <unordered_map>
#include <vector>

#include "device_types.h"
#include "parquet_meta.h"
#include "../../include/frostgpu.h"

namespace fgpu {

// Table-wide dictionary of one string column: chunk-local dictionary indices are translated to
// these ids at upload, so group keys compare as small integers across parts and row groups.
struct GlobalDict {
  std::vector<std::string> values;
  std::unordered_map<std::string, uint32_t> index;
  bool preloaded = false;  // fgpu_dict_preload named this column: it exists on some rank of a multi-GPU run
  uint32_t intern(const char* p, size_t n) {
    std::string s(p, n);
    auto it = index.find(s);
    if (it != index.end()) return it->second;
    uint32_t id = uint32_t(values.size());
    values.push_back(s);
    index.emplace(std::move(s), id);
    return id;
  }
  uint32_t cardinality() const { return uint32_t(values.size()); }
  const std::string& value(uint32_t id) const { return values[id]; }
};

// Chunk-local dictionary of one string chunk, in order of first occurrence, each new entry interned into the table's
// GlobalDict.  The host's one reference interner: Arrow string arrays, PLAIN string pages built without a device, and
// the distinct PLAIN values the device's intern batch found (fed in order of first occurrence, so the result is the
// same).  Keys alias the source bytes, which outlive the interner.
struct ChunkInterner {
  GlobalDict* gd;
  std::vector<uint32_t>* lut;  // chunk-local index -> global id
  std::vector<std::pair<std::string_view, uint32_t>> entries;  // dictionary page entries, hashed on the first add() only
  std::unordered_map<std::string_view, uint32_t> local;
  ChunkInterner(GlobalDict* g, std::vector<uint32_t>* l) : gd(g), lut(l) {}
  // a dictionary page entry: its own chunk-local index, numbered as the page numbers it
  void entry(const char* p, size_t n) {
    entries.push_back({std::string_view(p, n), uint32_t(lut->size())});
    lut->push_back(gd->intern(p, n));
  }
  // a value: its chunk-local index; a value not seen before is appended
  uint32_t add(const char* p, size_t n) {
    for (const auto& e : entries) local.emplace(e.first, e.second);  // (a repeated entry keeps its first index)
    entries.clear();
    const std::string_view s(p, n);
    auto it = local.find(s);
    if (it != local.end()) return it->second;
    const uint32_t idx = uint32_t(lut->size());
    local.emplace(s, idx);
    lut->push_back(gd->intern(p, n));
    return idx;
  }
};

struct ChunkHost {
  ChunkDesc desc{};            // device pointers (valid once the part is uploaded)
  int32_t phys = -1;           // Parquet physical type
  uint64_t stored_bytes = 0;   // algorithmic bytes: footer total_compressed_size, total_uncompressed_size with a codec
  int32_t codec = 0;           // Parquet compression codec of the chunk (0 or LZ4_RAW)
  uint32_t lz4_pages = 0;      // its pages whose values the device inflates at upload
  uint64_t meta_bytes = 0;     // directories / indexes / LUTs
  std::string error;           // non-empty: unreadable; an error only if a query projects it
  bool has_minmax = false;     // footer statistics of an INT64 / DOUBLE chunk (known before the column is built)
  int64_t min_bits = 0, max_bits = 0;
  int64_t null_count = -1;     // -1: not recorded
  bool has_minmax_str = false; // BYTE_ARRAY chunk: bounding strings of the non-null values
  std::string min_str, max_str;
  std::vector<uint8_t> bloom;      // split-block bloom filter of the chunk (copied out of the file at put; empty: none)
  std::vector<uint32_t> lut_host;  // CK_DICT_STR: chunk dictionary index -> *local* global id
  // section offsets inside the part image (patched into desc after upload)
  int64_t off_values = -1, off_runs = -1, off_seeds = -1, off_def = -1, off_def_runs = -1, off_def_seeds = -1, off_lut = -1,
          off_dict64 = -1;
  int64_t dev_seeds = -1, dev_def_seeds = -1;  // seeds derived on the device: offsets inside the image's device-only region
  int64_t off_row_runs = -1, off_row_seeds = -1, dev_row_seeds = -1;  // row-space directory of a nullable run-length column
  // flat code array of a CK_DICT_STR chunk (device pointer; derived on first use by k_flatten, see tile_agg.cu)
  const uint8_t* flat = nullptr;
  uint8_t flat_w = 0, flat_bias = 0;
  // frame-of-reference image of a dense (CK_PLAIN64) non-null INT64 chunk whose range fits 32 bits (device pointer; derived on first
  // use by the sorted-run kernel, see ensure_narrow): narrow_w bytes per row holding value - narrow_base
  const uint8_t* narrow = nullptr;
  uint8_t narrow_w = 0;
  int64_t narrow_base = 0;
  // exclusive prefix sums of a dense (CK_PLAIN64) non-null INT64 chunk, n_rows + 1 entries modulo 2^64 (device pointer; derived on
  // first use by the prefix path of the sorted-run scan, see ensure_narrow)
  const long long* prefix = nullptr;
};

struct RowGroupHost {
  uint32_t n_rows = 0;
  std::map<std::string, ChunkHost> cols;
};

// A byte range of the source Parquet file that is copied to the device as is (PLAIN value regions):
// no host-side copy is made, the H2D copy reads straight from the (ideally pinned) source buffer.
struct Extent {
  const uint8_t* src;
  uint64_t len;
  uint64_t dst_off;  // offset inside the column image
};

// One PLAIN, DELTA_LENGTH_BYTE_ARRAY or DELTA_BYTE_ARRAY page of a chunk: its values become one bit-packed run of
// chunk-local indices, whose payload is a hole in the value-stream section (zero until the indices are written into it).
struct StrPage {
  uint32_t run;       // its entry in the chunk's value directory
  uint32_t first, n;  // its non-null values: ordinals [first, first + n) among the chunk's non-dictionary values
  uint64_t hole = 0;  // once the sections are written: image offset of its ceil(n / 8) * w index bytes
};

// One DELTA_BYTE_ARRAY page of a chunk: values [v0, v0 + n) of the chunk, front-coded.  Value i is the first
// str_pre[d0 + i - v0] bytes of value i - 1 (of "" for the page's first value), then its suffix.
struct StrFront {
  uint32_t v0, d0, w0, n;  // first value; its index in str_pre / str_suf; the page's first window in str_wmin; values
};

// How the 8 * n bytes of one CK_PLAIN64 page's values reach the chunk's value array: copied from `src` as they are, or
// a hole the device fills at upload from a DELTA_BINARY_PACKED stream (delta_int64.cu) or by inflating an LZ4_RAW block
// (lz4_pages.cu).
enum ValueFill : uint8_t { FILL_COPY, FILL_DBP, FILL_LZ4 };

// One page of a CK_PLAIN64 chunk: its dense values [v0, v0 + n) among the chunk's values.
struct ValuePage {
  ValueFill fill;
  const uint8_t* src;   // COPY: the values; DBP: the encoded stream; LZ4: the block, validated by the page walk
  uint64_t len;         // bytes read from src (DBP: the stream's; what follows it in the page is not read)
  uint32_t v0, n;
  // DBP: the header's first value, values per miniblock, and its miniblocks holding values in the walk's (then the
  // image's) miniblock list
  int64_t first = 0;
  uint64_t per_mb = 0;
  uint32_t mb0 = 0, n_mb = 0;
  uint64_t hole = 0;    // DBP / LZ4, once the sections are written: image offset of its values
};

// What the page walk of one chunk leaves for the section writing (the two halves of building a column).
struct ChunkWalk {
  ChunkHost host;                 // footer facts, kind, error
  std::vector<uint8_t> defstream;
  std::vector<HostRun> defruns;
  std::vector<uint64_t> valid;    // bitset of the non-null rows (nullable chunks that are not all present)
  uint32_t n_values = 0;
  std::vector<uint8_t> vstream;   // dictionary-index pages, without the PLAIN pages' holes
  std::vector<HostRun> vruns;     // a PLAIN page's entry holds its hole's position in `vstream` until the holes exist
  std::vector<std::pair<const uint8_t*, uint32_t>> dict_entries;  // string dictionary page, validated
  std::vector<int64_t> dict64;
  std::vector<ValuePage> value_pages;  // pages of an int64 / double chunk, in file order
  std::vector<DbpMiniblock> dbp_mbs;   // its DBP pages' miniblocks holding values, `first` rebased onto the chunk's values
  // Non-dictionary string values (PLAIN, DELTA_LENGTH_BYTE_ARRAY, DELTA_BYTE_ARRAY pages), validated: every value lies
  // inside its page.  They are addressed in one 32-bit space per chunk: [0, str_span) the file bytes from str_base,
  // [str_rb0, str_rb0 + str_rebuilt_len) the DELTA_BYTE_ARRAY values rebuilt from their prefixes and suffixes.
  const uint8_t* str_base = nullptr;  // value region of the first non-dictionary page
  uint32_t str_span = 0;              // bytes from str_base to the end of the last non-dictionary page's value region
  std::vector<uint32_t> str_off;      // per value: str_len empty: offset of its 4-byte length prefix; else its start
  std::vector<uint32_t> str_len;      // per value: its length (empty while the chunk holds PLAIN pages only)
  std::vector<StrPage> str_pages;
  // DELTA_BYTE_ARRAY pages: per page, per value its prefix length and the start of its suffix (in the file bytes),
  // per window of 32 values of a page the least prefix length in it
  std::vector<StrFront> str_fronts;
  std::vector<uint32_t> str_pre, str_suf, str_wmin;
  uint32_t str_rb0 = 0xffffffffu;     // start of the rebuilt values (none: no value starts there)
  uint64_t str_rebuilt_len = 0;
  const uint8_t* str_rebuilt = nullptr;     // host bytes of the rebuilt region (all of it, or the values being interned)
  std::vector<uint8_t> str_rebuilt_host;    // the host's own rebuild (unfront_strings)
  // intern result: the first ordinal of every distinct value, ascending (left by the device's intern batch;
  // empty: the host interns row by row), and after the section writing the chunk-local index of each of them
  std::vector<uint32_t> str_firsts, str_codes;
  uint32_t str_w = 0;  // bit width of the non-dictionary pages' indices
};

// Non-dictionary string value `i` of a walked chunk (a rebuilt DELTA_BYTE_ARRAY value needs str_rebuilt).
inline std::string_view chunk_string(const ChunkWalk& wk, uint32_t i) {
  const uint32_t off = wk.str_off[i];
  if (wk.str_len.empty()) {
    const uint8_t* p = wk.str_base + off;
    uint32_t l;
    std::memcpy(&l, p, 4);
    return std::string_view(reinterpret_cast<const char*>(p + 4), l);
  }
  const uint8_t* p = off >= wk.str_rb0 ? wk.str_rebuilt + (off - wk.str_rb0) : wk.str_base + off;
  return std::string_view(reinterpret_cast<const char*>(p), wk.str_len[i]);
}

// Rebuilds a walked chunk's DELTA_BYTE_ARRAY values on the host (str_rebuilt_host; no-op without such pages).
void unfront_strings(ChunkWalk* wk);

// Host staging of one column image, kept until its upload has been synchronised (release_staging).
struct ImageStaging {
  std::vector<uint8_t> meta;  // everything that is not an extent
  std::vector<Extent> extents;
  // the value pages of every chunk whose values the device writes at upload (not FILL_COPY; hole: image offset), and
  // their miniblocks (ValuePage::mb0 indexes this list)
  std::vector<ValuePage> value_pages;
  std::vector<DbpMiniblock> dbp_mbs;
  std::vector<StrCodeJob> str_jobs;  // PLAIN string pages whose indices the device writes at upload (dst: image offset)
};

// The host's reference of the device's fills: writes the values of every page in s.value_pages into its hole of
// `image`, a host copy of the column image.
void fill_value_pages(const ImageStaging& s, uint8_t* image);

// Device residency of one column of one part (all its row groups in one allocation).
struct ColumnImage {
  bool walked = false;     // page walk done (`walks` holds it until the sections are written)
  bool device_seeds = false;
  std::vector<ChunkWalk> walks;  // per row group, between the walk and the section writing
  bool built = false;      // host side done (ChunkHosts filled, dictionary interned)
  bool resident = false;   // bytes are on the device
  void* dev = nullptr;
  uint64_t dev_bytes = 0;
  ImageStaging staging;
  uint64_t seed_jobs_off = 0;    // SeedJob[n_seed_jobs] inside the meta region (device-derived seeds)
  uint32_t n_seed_jobs = 0, max_seed_chunks = 0;
  std::string error;             // whole-column error (a chunk the engine cannot read)
  void* flat_dev = nullptr;      // flat code arrays of every row group of this column (one allocation) + the job table
  bool narrowed = false;         // ensure_narrow ran (narrow_dev stays null when no chunk fits 32 bits)
  void* narrow_dev = nullptr;    // frame-of-reference images of every narrowed chunk of this column (one allocation)
  bool prefixed = false;         // ensure_narrow built the prefix-sum images
  void* prefix_dev = nullptr;    // prefix-sum images of every PLAIN non-null INT64 chunk of this column (one allocation)
};

struct Part {
  uint64_t id = 0, tx = 0;
  const uint8_t* file = nullptr;    // source bytes: borrowed (caller keeps them alive) or `owned`
  uint64_t file_bytes = 0;
  std::vector<uint8_t> owned;
  bool borrowed = false;
  bool arrow = false;               // L0 Arrow record: LSM.Scan hands it to the plan unfiltered (index/lsm.go:420-427)
  ParsedFile pf;
  std::vector<RowGroupHost> rgs;
  std::vector<std::string> columns;  // schema order
  std::map<std::string, ColumnImage> images;
};

struct Table {
  uint64_t epoch = 0;  // changes whenever the set of parts or a dictionary does (0: not stamped yet); plans cache against it
  std::vector<std::unique_ptr<Part>> parts;  // insertion order
  std::map<std::string, GlobalDict> dicts;   // by column name
};

// Parses footer + page headers and prepares the row-group skeleton (no column is built yet).
bool open_part(const uint8_t* file, uint64_t len, Part* part, std::string* err);

// Builds the host side of one column of a part (no CUDA calls): run directories, seeds, dictionary
// LUTs into `image.staging.meta`, PLAIN value regions as extents.  Interns dictionary entries into `table`.
// ChunkDesc pointers are offsets until patch_column_pointers() is called.
// device_seeds: leave the cursor seeds to k_make_seeds (ColumnImage::seed_jobs_*) instead of building them here.
// PLAIN string pages are interned here on the host, row by row (ChunkInterner), and their indices packed by the host.
void build_column(int index_rows, Table* table, Part* part, const std::string& column, bool device_seeds = false);

// build_column in two halves, with the device's intern batch between them:
// walk_column walks every chunk's pages and validates them.  A column without PLAIN string values, or with an
// unreadable chunk, is finished at once (the host interns whatever PLAIN strings it has); otherwise it stays walked
// but not built, its ChunkWalks waiting for str_firsts.
void walk_column(int index_rows, Table* table, Part* part, const std::string& column, bool device_seeds);
// finish_column writes every chunk's sections.  host_intern == false: every chunk with PLAIN string values carries its
// str_firsts; their chunk-local indices come back in str_codes and the holes are left for the device (StrPage::hole).
// The walks are kept until the caller clears them.
void finish_column(int index_rows, Table* table, Part* part, const std::string& column, bool host_intern);

// The distinct strings of one column of a parsed Parquet file (pages walked), in the order a put of the file interns
// them: per row group the dictionary page, then the non-dictionary (PLAIN, DELTA_LENGTH_BYTE_ARRAY, DELTA_BYTE_ARRAY)
// pages' values not in it, in order of first occurrence.  Returns false on a chunk whose pages cannot be read.
bool column_dict_values(const ParsedFile& pf, const std::string& column, GlobalDict* out, std::string* err);

// L0 Arrow-record part (parts/arrow.go:14-55): one row group holding the record's rows.  Every column image
// is built here (the record is released by the caller afterwards): int64 / float64 arrays become PLAIN
// chunks (non-null values packed, the validity bitmap IS the bit-packed definition-level stream),
// dictionary<int, binary|utf8> and plain binary/utf8 arrays become dictionary chunks whose index stream is
// one 32-bit "bit-packed" run.  Returns false and sets err for unsupported layouts.
bool build_arrow_part(Table* table, Part* part, const ::ArrowSchema* schema, const ::ArrowArray* array, std::string* err);

// Patches device pointers into the column's ChunkDescs once the image lives at `dev_base`.
void patch_column_pointers(Part* part, const std::string& column, const uint8_t* dev_base);

// JSON description for fgpu_parquet_describe (host-only tests).
std::string describe_part_json(const uint8_t* file, uint64_t len, int tile_rows, std::string* err);

}  // namespace fgpu
