// Host-side Parquet reader for libfrostgpu: footer (Thrift compact), page walk, hybrid-run walk.
// Produces what the device needs to decode pages without touching Thrift: per column chunk the
// page payload extents, and per hybrid stream (dictionary indices, definition levels) a run
// directory.  Takes over the host half of pqarrow.ParquetConverter / parquet-go's page readers
// (reference: pqarrow/arrow.go:711-823 writeColumnToArray page loop; format facts SURVEY.md App. C).
#pragma once
#include <cstdint>
#include <string>
#include <vector>

namespace fgpu {

enum PhysType : int32_t {
  PT_BOOLEAN = 0, PT_INT32 = 1, PT_INT64 = 2, PT_INT96 = 3, PT_FLOAT = 4, PT_DOUBLE = 5,
  PT_BYTE_ARRAY = 6, PT_FIXED_LEN_BYTE_ARRAY = 7
};
enum PqEncoding : int32_t {
  ENC_PLAIN = 0, ENC_PLAIN_DICTIONARY = 2, ENC_RLE = 3, ENC_BIT_PACKED = 4,
  ENC_DELTA_BINARY_PACKED = 5, ENC_DELTA_LENGTH_BYTE_ARRAY = 6, ENC_DELTA_BYTE_ARRAY = 7,
  ENC_RLE_DICTIONARY = 8, ENC_BYTE_STREAM_SPLIT = 9
};
enum PageType : int32_t { PG_DATA = 0, PG_INDEX = 1, PG_DICTIONARY = 2, PG_DATA_V2 = 3 };

struct SchemaLeaf {
  std::string name;  // dotted path, e.g. "labels.job"
  int32_t phys = -1;
  int32_t max_def = 0;
  int32_t max_rep = 0;
  bool is_unsigned = false;  // converted type UINT_64 / logical INT(64,false)
};

struct PageInfo {
  int32_t type = 0;        // PG_DATA or PG_DATA_V2
  int32_t encoding = 0;    // of the values
  uint32_t num_values = 0; // rows in the page (flat columns), nulls included
  int64_t num_nulls = -1;  // -1: unknown (v1 page)
  const uint8_t* def = nullptr;  // RLE/bit-packed hybrid of definition levels (no length prefix)
  uint32_t def_len = 0;
  const uint8_t* values = nullptr;  // encoded values region
  uint32_t values_len = 0;
  // > 0: `values` is one LZ4_RAW block of `values_len` bytes (in the file) that inflates to `lz4_len` bytes of PLAIN
  // INT64 / DOUBLE values; the page walk has validated it, the device inflates it at upload (lz4_pages.cu)
  uint32_t lz4_len = 0;
};

struct ChunkMeta {
  int32_t leaf = -1;  // index into ParsedFile::leaves
  int32_t codec = 0;
  int64_t num_values = 0;
  int64_t total_compressed_size = 0;  // footer figure: the chunk's bytes in the file
  int64_t total_uncompressed_size = 0;  // footer figure: the same, pages inflated (== total_compressed_size without a codec)
  int64_t null_count = -1;            // from chunk statistics when present
  bool has_minmax = false;            // INT64 / DOUBLE chunks: footer statistics carry both bounds
  int64_t min_bits = 0, max_bits = 0; // raw 8-byte bounds of the non-null values
  bool has_minmax_str = false;        // BYTE_ARRAY chunks: both (possibly truncated, still bounding) strings recorded
  std::string min_str, max_str;
  // split-block bloom filter of the chunk (parquet-go writes one per sorting column, dynparquet/schema.go:1111-1157):
  // the bitset (aliases `file`), null when the chunk has none or it uses an algorithm / hash / compression other than
  // BLOCK / XXHASH / UNCOMPRESSED
  const uint8_t* bloom = nullptr;
  uint32_t bloom_bytes = 0;
  const uint8_t* dict = nullptr;      // dictionary page payload (PLAIN)
  uint32_t dict_len = 0;
  uint32_t dict_num_values = 0;
  std::vector<PageInfo> pages;
  // LZ4_RAW chunk: the pages the host inflates (dictionary page, then the data pages' values, or whole v1 pages of an
  // OPTIONAL column, in file order: one address space for a chunk's string values), kept as long as the file is parsed;
  // `dict` and the PageInfo pointers of these pages point into it
  std::vector<uint8_t> inflated;
  std::string error;  // non-empty: chunk is unreadable by this engine (reason); only an error if projected
  // page walk state: footers are parsed eagerly, page headers only for the chunks a query touches
  int64_t data_page_offset = -1, dict_page_offset = -1;
  bool pages_walked = false;
};

struct RowGroupMeta {
  int64_t num_rows = 0;
  std::vector<ChunkMeta> chunks;  // one per leaf, in leaf order
};

struct ParsedFile {
  std::vector<SchemaLeaf> leaves;
  std::vector<RowGroupMeta> row_groups;
  std::vector<std::pair<std::string, std::string>> kv;
  int64_t num_rows = 0;
  std::string created_by;
};

// Parses footer and walks every page header.  Pointers in the result alias `file`.
// Returns false and sets err on malformed input.
// With walk_pages == false only the footer is read; walk_chunk_pages() then fills a chunk on demand.
bool parse_parquet(const uint8_t* file, uint64_t len, ParsedFile* out, std::string* err, bool walk_pages = true);

// Walks the page headers of one column chunk (idempotent): fills pages / dict, or sets error.
void walk_chunk_pages(const uint8_t* file, uint64_t len, const SchemaLeaf& leaf, int64_t rg_rows, ChunkMeta* cm);

// XXH64 (the hash of Parquet bloom filters, seed 0 over the PLAIN encoding of the value: the 8 little-endian bytes of an
// INT64 / DOUBLE, the bytes of a BYTE_ARRAY without their length prefix).
uint64_t xxhash64(const uint8_t* data, size_t len, uint64_t seed);
// Split-block bloom filter check (Parquet format, BloomFilter.md): false = the value is definitely not in the chunk.
bool sbbf_check(const uint8_t* bitset, uint32_t bytes, uint64_t hash);
// Sets the bits of `hash` (the writer's half; used by the tests to build filters).
void sbbf_insert(uint8_t* bitset, uint32_t bytes, uint64_t hash);

// Parquet codecs (CompressionCodec): LZ4_RAW is the one the page walk inflates; every other non-zero codec is refused.
constexpr int32_t kCodecLz4Raw = 7;

// Parse step of one LZ4_RAW block (the LZ4 block format without a frame) that must inflate to exactly `out_len` bytes.
// Validates every sequence as liblz4's safe decoder does for an output buffer of `out_len` bytes, without writing any
// output: no literal run, length extension or offset runs past the block, no match offset is 0 or reaches before the
// start of the output, the output is exactly `out_len` bytes, the block ends right after a sequence without a match,
// and the end-of-block rules hold (a match may not start in the last 12 bytes of the output or the last 8 of the block,
// nor end in the last 5 bytes of the output; literal length extensions stop 15 bytes, match length extensions 4 bytes
// before the block's end).  An empty output is the block 0x00.
bool parse_lz4_raw(const uint8_t* src, uint64_t len, uint64_t out_len, std::string* err);
// Unpack step of a block the parse step accepted: its first `cap` (<= out_len) bytes into `dst`.
void unpack_lz4_raw(const uint8_t* src, uint64_t len, uint8_t* dst, uint64_t cap);

// One run of an RLE/bit-packed hybrid stream (Parquet "RLE" encoding).
struct HostRun {
  uint32_t start;  // ordinal of the run's first value within the chunk's value sequence
  uint32_t off;    // byte offset of the payload inside the chunk's concatenated stream section
  uint32_t val;    // RLE: the repeated value
  uint32_t meta;   // bit0: 1 = bit-packed, 0 = RLE; bits 8..15: bit width
};

// Walks one hybrid stream holding `count` values of width `w` (count clamps padded tails).
// Appends runs (start offsets relative to `start0`, payload offsets relative to `off0` + position
// in `data`).  Zero-length runs are never emitted.  Returns false on overrun/malformed input.
bool walk_hybrid(const uint8_t* data, uint32_t len, int w, uint32_t count, uint32_t start0,
                 uint32_t off0, std::vector<HostRun>* runs, std::string* err);

// Reads value i of a hybrid stream described by runs (host-side reference used by describe/tests).
uint32_t hybrid_value_at(const uint8_t* stream, const std::vector<HostRun>& runs, uint32_t ordinal, bool* was_rle = nullptr);

// One miniblock of a DELTA_BINARY_PACKED stream that holds values.
struct DbpMiniblock {
  uint64_t off;        // byte offset of its packed deltas from the stream's start
  uint64_t min_delta;  // its block's min delta, wrapped to the value type
  uint32_t first;      // ordinal of the value its first delta makes (>= 1: value 0 is the header's first value)
  uint32_t count;      // values it makes
  uint32_t width;      // bit width of its deltas
};

// What the parse step of a DELTA_BINARY_PACKED stream leaves: the header and the miniblocks holding values.
struct DbpStream {
  uint64_t first = 0;   // the first value, wrapped to the value type
  uint32_t count = 0;   // values in the stream
  uint64_t per_mb = 0;  // values per miniblock
  uint64_t used = 0;    // the stream's bytes (miniblocks holding values are whole; the unused ones of the last block are absent)
  std::vector<DbpMiniblock> mbs;
};

// Parse step of one DELTA_BINARY_PACKED stream of `count` values of type T, without unpacking a delta.  Validates the
// header (block size a multiple of 128, values per miniblock a multiple of 32, total == count), the bit width of every
// miniblock that holds values (<= the bits of T) and that no header, width list or miniblock (written whole) runs
// past `len`.
template <typename T>
bool parse_delta_binary_packed(const uint8_t* data, uint64_t len, uint32_t count, DbpStream* out, std::string* err);

// Unpack step: the values of the miniblocks `mbs[0, n_mbs)` of a parsed stream at `data`, with the format's wrap-around
// arithmetic.  out[0] = first; the deltas of a miniblock make out[mb.first - ord0, + mb.count) (ord0: 0 for a parse
// result, the page's first ordinal for miniblocks rebased onto a chunk's value ordinals).
template <typename T>
void unpack_delta_binary_packed(const uint8_t* data, T first, const DbpMiniblock* mbs, size_t n_mbs, uint32_t ord0, T* out);

// Parse and unpack step of one stream (int32_t: the length streams of DELTA_LENGTH_BYTE_ARRAY / DELTA_BYTE_ARRAY pages).
// `used`: DbpStream::used.
template <typename T>
bool decode_delta_binary_packed(const uint8_t* data, uint64_t len, uint32_t count, std::vector<T>* out, uint64_t* used, std::string* err);

}  // namespace fgpu
