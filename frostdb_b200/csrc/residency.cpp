// Column residency (residency.h): uploads of column images, the device's string intern batch, and the flat,
// frame-of-reference and prefix-sum images derived from resident columns.
#include "residency.h"

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cstring>
#include <limits>
#include <map>
#include <thread>

#include "kernels.h"

namespace fgpu {
namespace {

int32_t cuda_fail(const char* what, cudaError_t e) {
  cudaGetLastError();
  return fail(FGPU_ERR_CUDA, std::string(what) + cudaGetErrorString(e));
}

// Copies bytes the host assembled to the device on the engine stream, through the page-locked arena when it has room:
// a pageable source would make the copy wait for the transfers queued before it.
cudaError_t h2d(fgpu_ctx* ctx, void* dst, const void* src, size_t bytes) {
  if (void* pin = ctx->arena_take(bytes)) {
    std::memcpy(pin, src, bytes);
    src = pin;
  }
  return cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, ctx->stream);
}

// A source range; `last`: the transfer ends with it; `own`: it lies in a buffer of its own (host-inflated LZ4_RAW pages,
// not the part's file), so that it is a transfer of its own.
struct Range { const uint8_t* src; uint64_t len; bool last = false; bool own = false; };

bool outside_file(const Part* part, const uint8_t* p) { return p < part->file || p >= part->file + part->file_bytes; }
// One transfer of the source ranges [first, first + n); where it goes in the staging buffer is its caller's choice
// (kToImage: not in it).
constexpr uint64_t kToImage = ~uint64_t(0);
struct Span { const uint8_t* src; uint64_t len, stage_off; size_t first, n; };

// Source ranges in ascending order, neighbours a few page headers apart joined into one transfer.
std::vector<Span> coalesce(const std::vector<Range>& ranges) {
  constexpr uint64_t kGap = 4096;
  std::vector<Span> spans;
  bool closed = true;
  for (size_t i = 0; i < ranges.size(); i++) {
    const Range& r = ranges[i];
    const uint8_t* end = closed ? nullptr : spans.back().src + spans.back().len;
    if (end && !r.own && r.src >= end && uint64_t(r.src - end) <= kGap) {
      spans.back().len = uint64_t(r.src - spans.back().src) + r.len;
      spans.back().n++;
    } else {
      spans.push_back({r.src, r.len, kToImage, i, 1});
    }
    closed = r.last || r.own;
  }
  return spans;
}

uint64_t al16(uint64_t n) { return (n + 15) & ~uint64_t(15); }

// Device scratch of one intern batch (intern_plain_strings): the images of the columns it finished hold StrCodeJobs
// into it until their upload launches them.  Freed in stream order when the batch goes; a finished column whose
// jobs were never launched (its upload did not happen) is reset to unbuilt, so that it is interned again when needed.
struct StrBatch {
  DevBuf scratch;
  std::vector<std::pair<Part*, std::string>> cols;
  StrBatch() = default;
  StrBatch(const StrBatch&) = delete;
  StrBatch& operator=(const StrBatch&) = delete;
  ~StrBatch() {
    for (auto& [part, col] : cols) {
      ColumnImage& img = part->images[col];
      if (!img.staging.str_jobs.empty() && !img.resident) img = ColumnImage{};
    }
  }
};

// Non-dictionary string pages of every listed column that walk_column left walked but not built, interned on the device
// in one batch (intern_strings.cu): the chunks' value regions and value addresses go up with one transfer per contiguous
// span, k_str_unfront rebuilds the DELTA_BYTE_ARRAY values behind their chunk's file bytes, k_str_hash and k_str_compact
// leave every distinct value's first occurrence in page-locked memory, k_str_gather (batches with DELTA_BYTE_ARRAY
// values only) copies the distinct rebuilt values there too, and after the one synchronisation the host interns the
// new strings in order of first occurrence (finish_column), uploads the chunk-local index of every distinct value and
// queues one StrCodeJob per page on the column's image.
int32_t intern_plain_strings(fgpu_ctx* ctx, Table* table, const std::vector<std::pair<Part*, std::string>>& cols, StrBatch* batch) {
  struct Item {
    ChunkWalk* wk;
    Part* part;
    uint64_t v0, s0, cap, byte_off;
    uint64_t l0, d0, w0, r0;  // in the batch's lengths, prefix / suffix, window and rebuilt-value arrays
  };
  std::vector<Item> items;
  std::vector<std::pair<Part*, std::string>> todo;
  uint64_t nv = 0, ns = 0, nl = 0, nd = 0, nw = 0, nr = 0, n_fronts = 0;
  for (const auto& pc : cols) {
    ColumnImage& img = pc.first->images[pc.second];
    if (!img.walked || img.built) continue;
    todo.push_back(pc);
    for (ChunkWalk& wk : img.walks) {
      if (!wk.host.error.empty() || wk.str_off.empty()) continue;
      uint64_t cap = 16;
      while (cap < 2 * uint64_t(wk.str_off.size())) cap <<= 1;
      items.push_back({&wk, pc.first, nv, ns, cap, 0, nl, nd, nw, nr});
      nv += wk.str_off.size();
      ns += cap;
      nl += wk.str_len.size();
      nd += wk.str_pre.size();
      nw += wk.str_wmin.size();
      if (!wk.str_fronts.empty()) nr += (wk.str_rebuilt_len + 15) & ~uint64_t(15);
      for (const StrFront& f : wk.str_fronts) n_fronts += (f.n + kFrontSeg - 1) / kFrontSeg;
    }
  }
  if (todo.empty()) return FGPU_OK;
  batch->cols.insert(batch->cols.end(), todo.begin(), todo.end());
  if (ns > 0xffffffffull) return fail(FGPU_ERR_UNSUPPORTED, "PLAIN string values of one upload exceed 2^31");
  // value regions: neighbouring chunks' regions travel as one transfer, 16-byte aligned; a chunk with
  // DELTA_BYTE_ARRAY values ends its span, and its rebuilt values follow at str_rb0 from its first byte
  std::vector<Range> ranges;
  for (const Item& it : items)
    ranges.push_back({it.wk->str_base, it.wk->str_span, !it.wk->str_fronts.empty(), outside_file(it.part, it.wk->str_base)});
  std::vector<Span> spans = coalesce(ranges);
  uint64_t payload = 0;
  for (Span& sp : spans) {
    sp.stage_off = payload;
    for (size_t k = sp.first; k < sp.first + sp.n; k++) items[k].byte_off = sp.stage_off + uint64_t(items[k].wk->str_base - sp.src);
    const Item& last = items[sp.first + sp.n - 1];
    payload = last.wk->str_fronts.empty() ? sp.stage_off + al16(sp.len) : al16(last.byte_off + last.wk->str_rb0 + last.wk->str_rebuilt_len);
  }
  // scratch: [chunks][counts][offsets][lengths][prefixes][suffixes][windows][front jobs][slots][codes][first / rank][keys]
  // [payload], 16-byte aligned pieces (the pieces of delta pages are empty in a batch of PLAIN pages)
  const auto al = al16;
  const uint64_t n = items.size();
  const uint64_t o_cnt = al(n * sizeof(StrChunk)), o_off = o_cnt + al(n * 4), o_len = o_off + al(nv * 4), o_pre = o_len + al(nl * 4),
                 o_suf = o_pre + al(nd * 4), o_wmin = o_suf + al(nd * 4), o_jobs = o_wmin + al(nw * 4),
                 o_slot = o_jobs + al(n_fronts * sizeof(StrFrontJob)), o_code = o_slot + al(nv * 4), o_first = o_code + al(nv * 4),
                 o_keys = o_first + al(ns * 4), o_pay = o_keys + ns * 8;
  CUDA_TRY(batch->scratch.alloc(o_pay + payload, ctx->stream));
  uint8_t* d = static_cast<uint8_t*>(batch->scratch.p);
  // first occurrences (written by k_str_compact), counts, rebuilt regions (the distinct values written by k_str_gather)
  const uint64_t pin_rebuilt = al(nv * 4 + n * 4);
  const PinnedBlock pin_block(ctx->pinned, size_t(pin_rebuilt + nr));
  if (!pin_block) return fail(FGPU_ERR_OOM, "PLAIN string interning: page-locked result buffer");
  uint8_t* pin = pin_block.get();
  uint32_t* h_first = reinterpret_cast<uint32_t*>(pin);
  uint32_t* h_count = h_first + nv;
  std::vector<uint8_t> head(o_slot, 0);  // chunk table, zero counts, value addresses, front jobs
  uint64_t job = 0;
  for (size_t i = 0; i < items.size(); i++) {
    const Item& it = items[i];
    const ChunkWalk& wk = *it.wk;
    StrChunk c{};
    c.bytes = d + o_pay + it.byte_off;
    c.off = reinterpret_cast<const uint32_t*>(d + o_off) + it.v0;
    c.len = wk.str_len.empty() ? nullptr : reinterpret_cast<const uint32_t*>(d + o_len) + it.l0;
    c.keys = reinterpret_cast<unsigned long long*>(d + o_keys) + it.s0;
    c.first = reinterpret_cast<uint32_t*>(d + o_first) + it.s0;
    c.slot = reinterpret_cast<uint32_t*>(d + o_slot) + it.v0;
    c.out_first = h_first + it.v0;
    c.n = uint32_t(wk.str_off.size());
    c.mask = uint32_t(it.cap - 1);
    c.v0 = uint32_t(it.v0);
    c.s0 = uint32_t(it.s0);
    c.rb0 = wk.str_rb0;
    if (!wk.str_fronts.empty()) {
      c.pre = reinterpret_cast<const uint32_t*>(d + o_pre) + it.d0;
      c.suf = reinterpret_cast<const uint32_t*>(d + o_suf) + it.d0;
      c.wmin = reinterpret_cast<const uint32_t*>(d + o_wmin) + it.w0;
      c.out_rebuilt = pin + pin_rebuilt + it.r0;
      std::memcpy(head.data() + o_pre + it.d0 * 4, wk.str_pre.data(), wk.str_pre.size() * 4);
      std::memcpy(head.data() + o_suf + it.d0 * 4, wk.str_suf.data(), wk.str_suf.size() * 4);
      std::memcpy(head.data() + o_wmin + it.w0 * 4, wk.str_wmin.data(), wk.str_wmin.size() * 4);
      for (const StrFront& f : wk.str_fronts)
        for (uint32_t seg = 0; seg < f.n; seg += kFrontSeg) {
          const StrFrontJob fj{uint32_t(i), f.v0, f.d0, f.w0, seg, std::min(kFrontSeg, f.n - seg)};
          std::memcpy(head.data() + o_jobs + job++ * sizeof(StrFrontJob), &fj, sizeof fj);
        }
    }
    std::memcpy(head.data() + i * sizeof(StrChunk), &c, sizeof c);
    std::memcpy(head.data() + o_off + it.v0 * 4, wk.str_off.data(), wk.str_off.size() * 4);
    if (!wk.str_len.empty()) std::memcpy(head.data() + o_len + it.l0 * 4, wk.str_len.data(), wk.str_len.size() * 4);
  }
  cudaError_t e = h2d(ctx, d, head.data(), head.size());
  if (e == cudaSuccess) e = cudaMemsetAsync(d + o_first, 0xff, size_t(o_pay - o_first), ctx->stream);  // first = ~0, keys empty
  for (const Span& sp : spans) {
    if (e != cudaSuccess) break;
    e = cudaMemcpyAsync(d + o_pay + sp.stage_off, sp.src, sp.len, cudaMemcpyHostToDevice, ctx->stream);
  }
  const StrChunk* d_chunks = reinterpret_cast<const StrChunk*>(d);
  uint32_t* d_count = reinterpret_cast<uint32_t*>(d + o_cnt);
  if (e == cudaSuccess) e = launch_str_unfront(d_chunks, reinterpret_cast<const StrFrontJob*>(d + o_jobs), uint32_t(n_fronts), ctx->stream);
  if (e == cudaSuccess) e = launch_str_hash(d_chunks, uint32_t(n), uint32_t(nv), ctx->stream);
  if (e == cudaSuccess) e = launch_str_compact(d_chunks, uint32_t(n), uint32_t(ns), d_count, ctx->stream);
  if (e == cudaSuccess && nr > 0) e = launch_str_gather(d_chunks, uint32_t(n), uint32_t(ns), ctx->stream);
  if (e == cudaSuccess) e = cudaMemcpyAsync(h_count, d_count, n * 4, cudaMemcpyDeviceToHost, ctx->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
  if (e != cudaSuccess) return cuda_fail("PLAIN string interning: ", e);
  // first occurrences in ascending order (they name the distinct values), remembering each one's rank
  std::vector<std::vector<uint32_t>> rank_of(items.size());
  for (size_t i = 0; i < items.size(); i++) {
    const uint32_t cnt = h_count[i];
    std::vector<std::pair<uint32_t, uint32_t>> fr(cnt);
    for (uint32_t r = 0; r < cnt; r++) fr[r] = {h_first[items[i].v0 + r], r};
    std::sort(fr.begin(), fr.end());
    items[i].wk->str_firsts.resize(cnt);
    rank_of[i].resize(cnt);
    for (uint32_t k = 0; k < cnt; k++) {
      items[i].wk->str_firsts[k] = fr[k].first;
      rank_of[i][k] = fr[k].second;
    }
    if (!items[i].wk->str_fronts.empty()) items[i].wk->str_rebuilt = pin + pin_rebuilt + items[i].r0;
  }
  // the sections: interning of the new strings, holes for the indices; then the chunk-local index per rank
  std::vector<uint32_t> codes;
  std::vector<uint64_t> code0(items.size());
  for (const auto& [part, col] : todo) finish_column(kIndexRows, table, part, col, /*host_intern=*/false);
  for (size_t i = 0; i < items.size(); i++) {
    code0[i] = codes.size();
    codes.resize(codes.size() + rank_of[i].size());
    const ChunkWalk& wk = *items[i].wk;
    if (wk.str_codes.size() != rank_of[i].size()) continue;  // the chunk was refused while its sections were written
    for (size_t k = 0; k < rank_of[i].size(); k++) codes[code0[i] + rank_of[i][k]] = wk.str_codes[k];
  }
  if (!codes.empty()) e = h2d(ctx, d + o_code, codes.data(), codes.size() * 4);
  if (e != cudaSuccess) return cuda_fail("PLAIN string interning: ", e);
  size_t i = 0;
  for (const auto& [part, col] : todo) {
    ColumnImage& img = part->images[col];
    for (size_t g = 0; g < img.walks.size(); g++) {
      const ChunkWalk& wk = img.walks[g];
      if (i >= items.size() || items[i].wk != &wk) continue;
      const Item& it = items[i];
      const uint64_t c0 = code0[i++];
      if (!img.error.empty()) continue;  // a refused chunk makes the column unreadable: it is never uploaded
      for (const StrPage& pg : wk.str_pages) {
        StrCodeJob j{};
        j.dst = reinterpret_cast<uint8_t*>(uintptr_t(pg.hole));  // image offset: rebased at upload
        j.slot = reinterpret_cast<const uint32_t*>(d + o_slot) + it.v0 + pg.first;
        j.rank = reinterpret_cast<const uint32_t*>(d + o_first) + it.s0;
        j.code = reinterpret_cast<const uint32_t*>(d + o_code) + c0;
        j.n = pg.n;
        j.w = wk.str_w;
        img.staging.str_jobs.push_back(j);
      }
    }
    img.walks.clear();
  }
  return FGPU_OK;
}

// The PLAIN string pages' indices of a column whose image is now at `dev` (queued by intern_plain_strings).
cudaError_t launch_str_jobs(fgpu_ctx* ctx, std::vector<StrCodeJob>& jobs, void* dev) {
  if (jobs.empty()) return cudaSuccess;
  uint32_t groups = 0;
  for (StrCodeJob& j : jobs) {
    j.dst = static_cast<uint8_t*>(dev) + reinterpret_cast<uintptr_t>(j.dst);
    j.g0 = groups;
    groups += (j.n + 7) / 8;
  }
  DevBuf d_jobs;  // released in stream order
  cudaError_t e = d_jobs.alloc(jobs.size() * sizeof(StrCodeJob), ctx->stream);
  if (e == cudaSuccess) e = h2d(ctx, d_jobs.p, jobs.data(), jobs.size() * sizeof(StrCodeJob));
  if (e == cudaSuccess) e = launch_str_codes(static_cast<const StrCodeJob*>(d_jobs.p), uint32_t(jobs.size()), groups, ctx->stream);
  return e;
}

// Source ranges of one kind of page in ascending order, coalesced and placed in the staging buffer from `off`: each
// transfer 16-byte aligned with >= 16 pad bytes behind it.  direct: a transfer of one range is not placed (stage_off
// stays kToImage), it goes straight to its place in the image.  row(i, at): range i lies at `at` in the staging buffer.
// Returns the end of the last placed transfer's padding.
template <typename Row>
uint64_t place(const std::vector<Range>& ranges, uint64_t off, bool direct, std::vector<Span>* spans, Row row) {
  *spans = coalesce(ranges);
  for (Span& sp : *spans) {
    if (direct && sp.n == 1) continue;
    sp.stage_off = off;
    off += al16(sp.len) + 16;
    for (size_t i = sp.first; i < sp.first + sp.n; i++) row(i, sp.stage_off + uint64_t(ranges[i].src - sp.src));
  }
  return off;
}

// The staging buffer of one column upload, one piece per kind of page, each piece 16-byte aligned (a kind without pages
// takes no space), and the tables the kernels read from it:
// - PLAIN pages: neighbouring page payloads (separated by a page header) as one transfer, then the PageCopy table;
//   k_gather_pages copies them into the dense value array.  A payload without neighbours goes straight to its place.
// - DELTA_BINARY_PACKED pages: their streams, then the page and miniblock tables, then the decode's scratch.
// - LZ4_RAW PLAIN INT64 / DOUBLE pages: their blocks, then the job table.
// Ranges of different kinds are never joined into one transfer.
struct StagePlan {
  std::vector<Span> plain, dbp, lz4;
  std::vector<PageCopy> copies;
  std::vector<DbpPage> dbp_pages;
  std::vector<DbpMini> dbp_mbs;
  std::vector<Lz4Job> lz4_jobs;
  uint64_t n_groups = 0;  // 32-value groups of the DELTA_BINARY_PACKED decode
  uint64_t copies_off = 0, dbp_tab_off = 0, scratch_off = 0, lz4_tab_off = 0;
  uint64_t bytes = 0;     // of the buffer (0: nothing is staged)
};

StagePlan plan_stage(const Part* part, const ImageStaging& s, uint8_t* dev) {
  StagePlan p;
  std::vector<Range> ranges;
  auto range = [&](const uint8_t* src, uint64_t len) { ranges.push_back({src, len, false, outside_file(part, src)}); };
  for (const Extent& x : s.extents) range(x.src, x.len);
  p.copies_off = place(ranges, 0, /*direct=*/true, &p.plain, [&](size_t i, uint64_t at) {
    p.copies.push_back({at, s.extents[i].dst_off, s.extents[i].len});
  });
  uint64_t end = p.copies_off + p.copies.size() * sizeof(PageCopy);
  std::vector<const ValuePage*> dbp, lz4;  // the pages the device fills, per kind in image order
  for (const ValuePage& pg : s.value_pages) (pg.fill == FILL_DBP ? dbp : lz4).push_back(&pg);
  if (!dbp.empty()) {
    ranges.clear();
    for (const ValuePage* pg : dbp) range(pg->src, pg->len);
    p.dbp_tab_off = place(ranges, al16(end), false, &p.dbp, [&](size_t i, uint64_t at) {
      const ValuePage& d = *dbp[i];
      DbpPage pg{};
      pg.dst = reinterpret_cast<unsigned long long*>(dev + d.hole);
      pg.src = at;
      pg.first = static_cast<unsigned long long>(d.first);
      pg.n = d.n;
      pg.g0 = uint32_t(p.n_groups);
      pg.mb0 = uint32_t(p.dbp_mbs.size());
      pg.per_mb = uint32_t(std::min<uint64_t>(d.per_mb, 0xffffffffu));
      p.n_groups += (d.n + 31) / 32;
      for (uint32_t m = d.mb0; m < d.mb0 + d.n_mb; m++)
        p.dbp_mbs.push_back(DbpMini{s.dbp_mbs[m].min_delta, uint32_t(s.dbp_mbs[m].off), s.dbp_mbs[m].width});
      p.dbp_pages.push_back(pg);
    });
    p.scratch_off = al16(p.dbp_tab_off + p.dbp_pages.size() * sizeof(DbpPage) + p.dbp_mbs.size() * sizeof(DbpMini));
    end = p.scratch_off + dbp_scratch_bytes(uint32_t(p.n_groups));
  }
  if (!lz4.empty()) {
    ranges.clear();
    for (const ValuePage* pg : lz4) range(pg->src, pg->len);
    p.lz4_tab_off = place(ranges, al16(end), false, &p.lz4, [&](size_t i, uint64_t at) {
      p.lz4_jobs.push_back(Lz4Job{dev + lz4[i]->hole, at, uint32_t(lz4[i]->len), lz4[i]->n * 8});
    });
    end = p.lz4_tab_off + p.lz4_jobs.size() * sizeof(Lz4Job);
  }
  if (!p.copies.empty() || !dbp.empty() || !lz4.empty()) p.bytes = end;
  return p;
}

// Copies a planned staging buffer's tables and transfers and launches the kernels that read them, in order:
// k_gather_pages, the DELTA_BINARY_PACKED decode, k_lz4_pages.  copied: the bytes of every transfer and of the
// DELTA_BINARY_PACKED and LZ4_RAW tables.
cudaError_t stage_pages(fgpu_ctx* ctx, const StagePlan& p, const std::vector<Extent>& extents, uint8_t* dev, uint8_t* stage,
                        uint64_t* copied) {
  cudaError_t e = cudaSuccess;
  auto send = [&](const std::vector<Span>& spans) {
    for (const Span& sp : spans) {
      if (e != cudaSuccess) return;
      *copied += sp.len;
      uint8_t* dst = sp.stage_off == kToImage ? dev + extents[sp.first].dst_off : stage + sp.stage_off;
      e = cudaMemcpyAsync(dst, sp.src, sp.len, cudaMemcpyHostToDevice, ctx->stream);
    }
  };
  if (!p.copies.empty()) e = h2d(ctx, stage + p.copies_off, p.copies.data(), p.copies.size() * sizeof(PageCopy));
  send(p.plain);
  if (e == cudaSuccess && !p.copies.empty())
    e = launch_gather_pages(stage, dev, reinterpret_cast<const PageCopy*>(stage + p.copies_off), uint32_t(p.copies.size()), ctx->stream);
  if (e == cudaSuccess && !p.dbp_pages.empty()) {
    const size_t pages = p.dbp_pages.size() * sizeof(DbpPage);
    std::vector<uint8_t> tab(pages + p.dbp_mbs.size() * sizeof(DbpMini));
    std::memcpy(tab.data(), p.dbp_pages.data(), pages);
    std::memcpy(tab.data() + pages, p.dbp_mbs.data(), tab.size() - pages);
    e = h2d(ctx, stage + p.dbp_tab_off, tab.data(), tab.size());
    *copied += tab.size();
    send(p.dbp);
    if (e == cudaSuccess)
      e = launch_dbp_decode(stage, reinterpret_cast<const DbpPage*>(stage + p.dbp_tab_off), uint32_t(p.dbp_pages.size()),
                            reinterpret_cast<const DbpMini*>(stage + p.dbp_tab_off + pages), uint32_t(p.n_groups),
                            stage + p.scratch_off, ctx->stream);
  }
  if (e == cudaSuccess && !p.lz4_jobs.empty()) {
    e = h2d(ctx, stage + p.lz4_tab_off, p.lz4_jobs.data(), p.lz4_jobs.size() * sizeof(Lz4Job));
    *copied += p.lz4_jobs.size() * sizeof(Lz4Job);
    send(p.lz4);
    if (e == cudaSuccess) e = launch_lz4_pages(stage, reinterpret_cast<const Lz4Job*>(stage + p.lz4_tab_off), uint32_t(p.lz4_jobs.size()), ctx->stream);
  }
  return e;
}

// Uploads one built column of one part if it is not resident yet: the host-assembled meta region with one copy, the
// pages' value bytes straight from the source file (or from the host-inflated pages of an LZ4_RAW chunk) through one
// staging allocation, then the string pages' indices and the cursor seeds, all on the engine stream so that kernels
// queued behind need no extra synchronisation.
int32_t upload_column(fgpu_ctx* ctx, Part* part, const std::string& column, uint64_t* h2d_bytes) {
  ColumnImage& img = part->images[column];
  if (!img.error.empty()) return FGPU_OK;  // surfaces as an error only if a query projects the column
  if (img.resident) return FGPU_OK;
  ImageStaging& s = img.staging;
  void* dev = nullptr;
  CUDA_TRY(cudaMallocAsync(&dev, img.dev_bytes, ctx->stream));
  uint8_t* d = static_cast<uint8_t*>(dev);
  cudaError_t e = h2d(ctx, dev, s.meta.data(), s.meta.size());
  uint64_t copied = s.meta.size();
  {
    const StagePlan plan = plan_stage(part, s, d);
    if (plan.n_groups > 0xffffffffull) e = cudaErrorInvalidValue;  // (more than 2^37 values in one column of one part)
    DevBuf stage;  // released in stream order when it goes out of scope
    if (plan.bytes && e == cudaSuccess) e = stage.alloc(plan.bytes, ctx->stream);
    if (e == cudaSuccess) e = stage_pages(ctx, plan, s.extents, d, static_cast<uint8_t*>(stage.p), &copied);
  }
  if (e == cudaSuccess) e = launch_str_jobs(ctx, s.str_jobs, dev);
  if (e == cudaSuccess) e = launch_make_seeds(dev, img.seed_jobs_off, img.n_seed_jobs, img.max_seed_chunks, ctx->stream);
  if (e != cudaSuccess) {
    cudaFreeAsync(dev, ctx->stream);
    return cuda_fail("column upload: ", e);
  }
  img.dev = dev;
  img.resident = true;
  patch_column_pointers(part, column, d);
  *h2d_bytes += copied;
  ctx->pending_uploads.push_back(&img);
  return FGPU_OK;
}

// Host side of several columns of one part in parallel (page walk, run directories, dictionary interning): the
// columns are independent — every column has its own dictionary, image and chunk records, all created here
// before the workers start so that no container is resized concurrently.
void prebuild_columns(Table* table, Part* part, const std::vector<std::string>& columns) {
  std::vector<const std::string*> todo;
  for (const std::string& c : columns) {
    ColumnImage& img = part->images[c];  // creates the entry
    if (img.built) continue;
    for (const SchemaLeaf& l : part->pf.leaves)
      if (l.name == c && l.phys == PT_BYTE_ARRAY) (void)table->dicts[c];
    todo.push_back(&c);
  }
  if (todo.size() < 2) return;  // a single column is built by its caller
  unsigned hw = std::thread::hardware_concurrency();
  const size_t n_threads = std::min<size_t>(todo.size(), std::min<size_t>(hw ? hw : 4, 32));  // (a part has ~20 columns: one wave)
  std::atomic<size_t> next{0};
  std::vector<std::thread> workers;
  for (size_t t = 0; t < n_threads; t++)
    workers.emplace_back([&]() {
      for (;;) {
        const size_t i = next.fetch_add(1);
        if (i >= todo.size()) break;
        walk_column(kIndexRows, table, part, *todo[i], /*device_seeds=*/true);  // (PLAIN strings: finished after the intern batch)
      }
    });
  for (std::thread& w : workers) w.join();
}

}  // namespace

int32_t upload_columns(fgpu_ctx* ctx, Table* table, const std::vector<std::pair<Part*, std::string>>& cols, UploadStats* st,
                       bool refuse_unreadable) {
  using Clock = std::chrono::steady_clock;
  auto since = [](Clock::time_point t) { return std::chrono::duration<double, std::micro>(Clock::now() - t).count(); };
  auto upload = [&](Part* part, const std::string& name) -> int32_t {
    const auto t = Clock::now();
    const int32_t rc = upload_column(ctx, part, name, &st->h2d_bytes);
    st->enqueue_us += since(t);
    if (rc) return rc;
    const ColumnImage& img = part->images[name];
    if (refuse_unreadable && !img.error.empty()) return fail(FGPU_ERR_UNSUPPORTED, "column " + name + ": " + img.error);
    return FGPU_OK;
  };
  StrBatch batch;
  auto t = Clock::now();
  int32_t rc = intern_plain_strings(ctx, table, cols, &batch);
  st->build_us += since(t);
  if (rc) return rc;
  std::vector<std::pair<Part*, std::string>> deferred;  // walked, waiting for the second intern batch
  for (const auto& [part, name] : cols) {
    t = Clock::now();
    walk_column(kIndexRows, table, part, name, /*device_seeds=*/true);
    st->build_us += since(t);
    if (!part->images[name].built) deferred.push_back({part, name});
    else if ((rc = upload(part, name))) return rc;
  }
  if (deferred.empty()) return FGPU_OK;
  t = Clock::now();
  rc = intern_plain_strings(ctx, table, deferred, &batch);
  st->build_us += since(t);
  if (rc) return rc;
  for (const auto& [part, name] : deferred)
    if ((rc = upload(part, name))) return rc;
  return FGPU_OK;
}

int32_t upload_part(fgpu_ctx* ctx, Table* table, Part* part) {
  prebuild_columns(table, part, part->columns);
  std::vector<std::pair<Part*, std::string>> cols;
  for (const std::string& col : part->columns) cols.push_back({part, col});
  UploadStats st;
  int32_t rc = upload_columns(ctx, table, cols, &st, /*refuse_unreadable=*/false);
  if (rc == FGPU_OK) {
    const cudaError_t e = cudaStreamSynchronize(ctx->stream);
    release_staging(ctx);
    if (e != cudaSuccess) rc = fail(FGPU_ERR_CUDA, std::string("part upload: ") + cudaGetErrorString(e));
  }
  if (rc) free_part(ctx, part);
  return rc;
}

int32_t ensure_flat(fgpu_ctx* ctx, Part* part, const std::string& column) {
  ColumnImage& img = part->images[column];
  if (img.flat_dev) return FGPU_OK;
  if (!img.resident) return fail(FGPU_ERR_INVALID, "flat codes requested for a column that is not resident: " + column);
  std::vector<FlatJob> jobs;
  std::vector<ChunkHost*> chs;
  std::vector<uint64_t> offs;
  uint64_t bytes = 0;
  uint32_t blocks = 0;
  for (RowGroupHost& rg : part->rgs) {
    auto it = rg.cols.find(column);
    if (it == rg.cols.end()) continue;
    ChunkHost& ch = it->second;
    if (!ch.error.empty() || ch.desc.kind != CK_DICT_STR) continue;
    uint32_t max_gid = 0;
    for (uint32_t g : ch.lut_host) max_gid = std::max(max_gid, g);
    FlatJob j{};
    j.chunk = ch.desc;
    j.bias = ch.desc.has_nulls ? 0u : 1u;
    const int bits = bit_width_u32(uint64_t(max_gid) + 1u - j.bias);
    j.w = bits <= 8 ? 8u : (bits <= 16 ? 16u : 32u);  // byte-aligned codes: one shared-memory load per row and column
    j.first_block = blocks;
    const uint32_t nb = (rg.n_rows + uint32_t(kIndexRows) - 1) / uint32_t(kIndexRows);
    blocks += nb;
    offs.push_back(bytes);
    bytes += (uint64_t(nb) * (kIndexRows / 8) * j.w + 64 + 127) & ~uint64_t(127);
    jobs.push_back(j);
    chs.push_back(&ch);
  }
  if (jobs.empty()) return FGPU_OK;
  void* dev = nullptr;
  CUDA_TRY(cudaMallocAsync(&dev, bytes + jobs.size() * sizeof(FlatJob), ctx->stream));
  for (size_t i = 0; i < jobs.size(); i++) jobs[i].out = static_cast<uint8_t*>(dev) + offs[i];
  FlatJob* d_jobs = reinterpret_cast<FlatJob*>(static_cast<uint8_t*>(dev) + bytes);
  cudaError_t e = h2d(ctx, d_jobs, jobs.data(), jobs.size() * sizeof(FlatJob));
  if (e == cudaSuccess) e = launch_flatten(d_jobs, uint32_t(jobs.size()), blocks, ctx->sm_count, ctx->stream);
  if (e != cudaSuccess) {
    cudaFreeAsync(dev, ctx->stream);
    return cuda_fail("flat codes: ", e);
  }
  img.flat_dev = dev;
  for (size_t i = 0; i < jobs.size(); i++) {
    chs[i]->flat = jobs[i].out;
    chs[i]->flat_w = uint8_t(jobs[i].w);
    chs[i]->flat_bias = uint8_t(jobs[i].bias);
  }
  return FGPU_OK;
}

// Frame-of-reference images of PLAIN non-null INT64 columns for the sorted-run kernel: for every resident chunk of every
// listed (part, column) whose range max - min fits 32 bits, one image of uint{8,16,32}(value - min) per row, the
// narrowest of the three (one allocation per (part, column), kept until the part goes).  The sorted-run kernel then
// stages 1, 2 or 4 bytes per row instead of 8.  Minimum and maximum come from the values on the device, not from the
// footer statistics, so that a chunk without statistics narrows as well and wrong statistics cannot change a result.
// The whole list costs one min / max launch, one synchronisation and one narrowing launch.
// want_prefix: (part, column) pairs that also get exclusive prefix-sum images for the prefix path of the sorted-run scan
// (k_runs_prefix): every PLAIN non-null INT64 chunk, whatever its range, n_rows + 1 wrapping int64 sums (one allocation
// per (part, column), kept until the part goes).  They are written by the same two launches: the min / max pass also
// leaves every block's sum, the narrowing pass turns the values into the prefix, so the values are read no more often.
int32_t ensure_narrow(fgpu_ctx* ctx, const std::vector<std::pair<Part*, std::string>>& want,
                      const std::vector<std::pair<Part*, std::string>>& want_prefix) {
  struct Job {
    ColumnImage* img;
    ChunkHost* ch;
    bool narrow, prefix;
  };
  std::vector<Job> host;
  std::vector<NarrowJob> jobs;
  std::vector<ColumnImage*> imgs, pimgs;
  uint32_t blocks = 0;
  std::map<std::pair<Part*, std::string>, std::pair<bool, bool>> todo;  // (narrow, prefix), in a fixed order
  for (const auto& pc : want) todo[pc].first = true;
  for (const auto& pc : want_prefix) todo[pc].second = true;
  for (const auto& kv : todo) {
    Part* part = kv.first.first;
    const std::string& col = kv.first.second;
    ColumnImage& img = part->images[col];
    const bool nar = kv.second.first && !img.narrowed, pre = kv.second.second && !img.prefixed;
    if (!nar && !pre) continue;
    if (!img.resident) return fail(FGPU_ERR_INVALID, "narrow image requested for a column that is not resident: " + col);
    if (nar) {
      img.narrowed = true;
      imgs.push_back(&img);
    }
    if (pre) {
      img.prefixed = true;
      pimgs.push_back(&img);
    }
    for (RowGroupHost& rg : part->rgs) {
      auto it = rg.cols.find(col);
      if (it == rg.cols.end()) continue;
      ChunkHost& ch = it->second;
      if (!ch.error.empty() || ch.desc.kind != CK_PLAIN64 || ch.desc.has_nulls || ch.phys != PT_INT64 || rg.n_rows == 0) continue;
      NarrowJob j{};
      j.src = reinterpret_cast<const long long*>(ch.desc.values);
      j.n_rows = rg.n_rows;
      j.first_block = blocks;
      j.sum_block = blocks;
      blocks += (rg.n_rows + kNarrowRows - 1) / kNarrowRows;
      jobs.push_back(j);
      host.push_back({&img, &ch, nar, pre});
    }
  }
  if (jobs.empty()) return FGPU_OK;
  const size_t jb = jobs.size() * sizeof(NarrowJob), mmb = jobs.size() * 16;
  std::vector<long long> mm(2 * jobs.size());
  for (size_t i = 0; i < jobs.size(); i++) {
    mm[2 * i] = std::numeric_limits<long long>::max();
    mm[2 * i + 1] = std::numeric_limits<long long>::min();
  }
  void* tmp = nullptr;  // [jobs][min, max per job][sum per block]
  CUDA_TRY(cudaMallocAsync(&tmp, jb + mmb + size_t(blocks) * 8, ctx->stream));
  NarrowJob* d_jobs = static_cast<NarrowJob*>(tmp);
  long long* d_mm = reinterpret_cast<long long*>(static_cast<uint8_t*>(tmp) + jb);
  unsigned long long* d_bsum = reinterpret_cast<unsigned long long*>(static_cast<uint8_t*>(tmp) + jb + mmb);
  cudaError_t e = h2d(ctx, d_jobs, jobs.data(), jb);
  if (e == cudaSuccess) e = h2d(ctx, d_mm, mm.data(), mmb);
  if (e == cudaSuccess) e = launch_chunk_minmax(d_jobs, uint32_t(jobs.size()), blocks, d_mm, d_bsum, ctx->stream);
  if (e == cudaSuccess) e = cudaMemcpyAsync(mm.data(), d_mm, mmb, cudaMemcpyDeviceToHost, ctx->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
  // widths, then one image allocation per (part, column) and the narrowing pass over the chunks that fit 32 bits or want
  // a prefix image
  std::map<ColumnImage*, uint64_t> bytes, pbytes;
  std::vector<uint64_t> offs(jobs.size()), poffs(jobs.size());
  std::vector<NarrowJob> pass2;
  uint32_t blocks2 = 0;
  for (size_t i = 0; i < jobs.size() && e == cudaSuccess; i++) {
    if (host[i].prefix) {
      uint64_t& b = pbytes[host[i].img];
      poffs[i] = b;
      b += (uint64_t(jobs[i].n_rows + 1) * 8 + 127) & ~uint64_t(127);
    }
    const uint64_t range = uint64_t(mm[2 * i + 1]) - uint64_t(mm[2 * i]);
    jobs[i].w = !host[i].narrow ? 0u : range <= 0xffu ? 1u : (range <= 0xffffu ? 2u : (range <= 0xffffffffu ? 4u : 0u));
    if (!jobs[i].w) continue;  // needs 64 bits: read from the extent as before
    jobs[i].base = mm[2 * i];
    uint64_t& b = bytes[host[i].img];
    offs[i] = b;
    b += (uint64_t(jobs[i].n_rows) * jobs[i].w + 16 + 127) & ~uint64_t(127);  // 128-byte aligned, >= 16 readable pad bytes (tile copies round up to 16)
  }
  for (ColumnImage* img : imgs) {
    auto it = bytes.find(img);
    if (it == bytes.end() || e != cudaSuccess) continue;
    e = cudaMallocAsync(&img->narrow_dev, it->second, ctx->stream);
  }
  for (ColumnImage* img : pimgs) {
    auto it = pbytes.find(img);
    if (it == pbytes.end() || e != cudaSuccess) continue;
    e = cudaMallocAsync(&img->prefix_dev, it->second, ctx->stream);
  }
  for (size_t i = 0; i < jobs.size() && e == cudaSuccess; i++) {
    if (jobs[i].w) jobs[i].out = static_cast<uint8_t*>(host[i].img->narrow_dev) + offs[i];
    if (host[i].prefix) jobs[i].pre = reinterpret_cast<long long*>(static_cast<uint8_t*>(host[i].img->prefix_dev) + poffs[i]);
    if (!jobs[i].w && !jobs[i].pre) continue;
    jobs[i].first_block = blocks2;
    blocks2 += (jobs[i].n_rows + kNarrowRows - 1) / kNarrowRows;
    pass2.push_back(jobs[i]);
  }
  if (e == cudaSuccess && !pass2.empty()) e = h2d(ctx, d_jobs, pass2.data(), pass2.size() * sizeof(NarrowJob));
  if (e == cudaSuccess) e = launch_narrow(d_jobs, uint32_t(pass2.size()), blocks2, d_bsum, ctx->stream);
  cudaFreeAsync(tmp, ctx->stream);
  if (e != cudaSuccess) return cuda_fail("narrow images: ", e);
  for (size_t i = 0; i < jobs.size(); i++) {
    if (jobs[i].pre) host[i].ch->prefix = jobs[i].pre;
    if (!jobs[i].w) continue;
    host[i].ch->narrow = jobs[i].out;
    host[i].ch->narrow_w = uint8_t(jobs[i].w);
    host[i].ch->narrow_base = jobs[i].base;
  }
  return FGPU_OK;
}

void release_staging(fgpu_ctx* ctx) {
  ctx->arena_used = 0;
  for (ColumnImage* img : ctx->pending_uploads) img->staging = ImageStaging{};
  ctx->pending_uploads.clear();
}

void free_part(fgpu_ctx* ctx, Part* p) {
  for (auto& kv : p->images) {
    if (kv.second.dev) cudaFreeAsync(kv.second.dev, ctx->stream);
    if (kv.second.flat_dev) cudaFreeAsync(kv.second.flat_dev, ctx->stream);
    if (kv.second.narrow_dev) cudaFreeAsync(kv.second.narrow_dev, ctx->stream);
    if (kv.second.prefix_dev) cudaFreeAsync(kv.second.prefix_dev, ctx->stream);
  }
}

}  // namespace fgpu
