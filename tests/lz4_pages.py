"""Parquet parts whose column chunks are LZ4_RAW-compressed (codec 7), each with an uncompressed twin holding the same
rows, and LZ4 blocks assembled by hand.

- Numeric layouts written by pyarrow through `dp.write_part` with every column LZ4_RAW (`ColumnDefinition.compression`):
  numeric_edges' INT_CHUNKS sorted and unsorted, an OPTIONAL `value` with an all-NULL page and an all-NULL row group
  (v1 and v2), data page v1 and v2, small pages with row groups of 4 096 + 7 rows, and DELTA_BINARY_PACKED `timestamp` /
  `value` under LZ4_RAW.
- String layouts (tests/plain_strings.py and tests/delta_strings.py rows): dictionary, dictionary falling back to PLAIN,
  PLAIN, DELTA_LENGTH_BYTE_ARRAY and DELTA_BYTE_ARRAY, v1 and v2.
- An LZ4 block writer driven by sequence plans: a plan is a list of (literal bytes, match or None), a match an (offset,
  length) pair; executing the plan gives the output, encoding it gives the block.  Every valid block is checked against
  pyarrow's decoder (`pa.Codec("lz4_raw")`), an independent implementation, when the set is built.
- A page-level writer that puts blocks into PLAIN INT64 pages (v1 and v2), a v2 page stored uncompressed in an LZ4_RAW
  chunk, and a compressed dictionary page; and a malformed set, one block per rule, with whether pyarrow takes it."""
import dataclasses
import functools
import io
import struct
from typing import Callable, Dict, List, Optional, Tuple

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq

from frostdb_b200 import dynparquet as dp
from tests import delta_int64 as di
from tests import delta_strings as ds
from tests import numeric_edges as ne
from tests import plain_strings as ps
from tests.delta_strings import _uleb, _zigzag
from tests.hybrid_pages import _Struct, bp, encode_hybrid

CK_PLAIN64, CK_DICT_STR = 1, 2
CODEC_LZ4_RAW = 7
LZ4 = pa.Codec("lz4_raw")


# ---- numeric layouts ---------------------------------------------------------------------------------------------
@dataclasses.dataclass(frozen=True)
class Layout:
    name: str
    make: Callable[[], Dict[str, object]]
    rg: int = ne.RG
    version: str = "2.0"
    data_page_size: Optional[int] = None
    nullable: bool = False
    delta: bool = False


LAYOUTS = [
    Layout("sorted", lambda: ne.int_part(ne.INT_CHUNKS, 301, sort=True)),
    Layout("unsorted", lambda: ne.int_part(ne.INT_CHUNKS, 302, sort=False)),
    Layout("sorted_v1", lambda: ne.int_part(ne.INT_CHUNKS, 303, sort=True), version="1.0"),
    Layout("nullable", lambda: di._nullable(304, ne.RG), data_page_size=2048, nullable=True),
    Layout("nullable_v1", lambda: di._nullable(305, ne.RG), version="1.0", data_page_size=2048, nullable=True),
    Layout("page_edges", lambda: ne.int_part(ne.INT_CHUNKS, 306, sort=True, rg=ne.RG + 7), rg=ne.RG + 7, data_page_size=512),
    Layout("page_edges_v1", lambda: ne.int_part(ne.INT_CHUNKS[:3], 307, sort=False, rg=ne.RG + 7), rg=ne.RG + 7, version="1.0",
           data_page_size=700),
    Layout("delta", lambda: ne.int_part(ne.INT_CHUNKS, 308, sort=True), delta=True),
    Layout("delta_nullable_v1", lambda: di._nullable(309, ne.RG), version="1.0", data_page_size=2048, nullable=True, delta=True),
]
LAYOUT_BY_NAME = {l.name: l for l in LAYOUTS}
NAMES = [l.name for l in LAYOUTS]


def schema(name: str, *, lz4: bool) -> dp.Schema:
    """numeric_edges' schema for the layout, every column LZ4_RAW when `lz4`."""
    l = LAYOUT_BY_NAME[name]
    s = di.schema(columns(name), delta=l.delta, nullable_value=l.nullable)
    for c in s.columns:
        c.compression = "LZ4_RAW" if lz4 else "NONE"
    return s


@functools.lru_cache(maxsize=None)
def columns(name: str) -> Dict[str, object]:
    """The layout's columns, without numeric_edges' `floatvalue` (its NaNs have no JSON form in a description)."""
    cols = LAYOUT_BY_NAME[name].make()
    cols.pop("floatvalue", None)
    return cols


def _write(name: str, lz4: bool) -> bytes:
    l = LAYOUT_BY_NAME[name]
    kwargs = {} if l.data_page_size is None else {"data_page_size": l.data_page_size}
    return dp.write_part(schema(name, lz4=lz4), columns(name), sort=False, row_group_size=l.rg, data_page_version=l.version, **kwargs)


@functools.lru_cache(maxsize=None)
def file_of(name: str) -> bytes:
    """The layout with every column LZ4_RAW."""
    return _write(name, True)


@functools.lru_cache(maxsize=None)
def twin_of(name: str) -> bytes:
    """The same rows, uncompressed."""
    return _write(name, False)


def codecs(buf: bytes) -> Dict[str, set]:
    """Per column, the codecs its chunks name."""
    md = pq.ParquetFile(io.BytesIO(buf)).metadata
    out = {}
    for g in range(md.num_row_groups):
        for j in range(md.num_columns):
            c = md.row_group(g).column(j)
            out.setdefault(c.path_in_schema, set()).add(c.compression)
    return out


def footer_sizes(buf: bytes, column: str) -> Tuple[int, int]:
    """(total_compressed_size, total_uncompressed_size) of `column` over the row groups."""
    md = pq.ParquetFile(io.BytesIO(buf)).metadata
    names = [md.schema.column(i).path for i in range(md.num_columns)]
    j = names.index(column)
    cs = [md.row_group(g).column(j) for g in range(md.num_row_groups)]
    return sum(c.total_compressed_size for c in cs), sum(c.total_uncompressed_size for c in cs)


def bytes_schema(lz4: bool) -> dp.Schema:
    """The reference's logictest `bytes` schema (logictest/logic_test.go:110-142) with `value` LZ4_RAW when `lz4`, as
    upstream stores it (dp.BytesDefinition itself stays uncompressed)."""
    s = dp.BytesDefinition()
    for c in s.columns:
        if c.name == "value" and lz4:
            c.compression = "LZ4_RAW"
    return s


# ---- string layouts ----------------------------------------------------------------------------------------------
# name -> (rows of tests/plain_strings.py or tests/delta_strings.py, how `s` is written)
STR_CASES = {
    "dict_v2": ("v2_optional", "dict"),
    "fallback_v1": ("fallback_v1", "fallback"),
    "fallback_v2": ("fallback_v2", "fallback"),
    "plain_v1": ("v1_optional", "plain"),
    "plain_v2": ("v2_optional", "plain"),
    "dlba_v1": ("v1_required", "dlba"),
    "dlba_v2": ("many_small_pages", "dlba"),
    "dba_v2": ("v2_optional", "dba"),
    "dba_front": (ds.FRONTS[0].name, "dba"),
}
STR_NAMES = list(STR_CASES)


def _str_write(name: str, lz4: bool, how: Optional[str] = None) -> bytes:
    rows, enc = STR_CASES[name]
    how = how or enc
    if rows in ds.FRONT_BY_NAME:
        f = ds.FRONT_BY_NAME[rows]
        version, rg, page, batch = f.version, f.n_rows, f.data_page_size, f.write_batch_size
    else:
        l = ps.LAYOUT_BY_NAME[rows]
        version, rg, page, batch = l.version, l.row_group_size or max(l.n_rows, 1), l.data_page_size, l.write_batch_size
    kwargs = {}
    if page is not None:
        kwargs["data_page_size"] = page
    if batch is not None:
        kwargs["write_batch_size"] = batch
    if how == "dict":
        kwargs.update(use_dictionary=["s"], dictionary_pagesize_limit=1 << 28)
    elif how == "fallback":
        kwargs.update(use_dictionary=["s"], dictionary_pagesize_limit=4096)
    else:
        kwargs["use_dictionary"] = False
        if how in ds.ENCODINGS:
            kwargs["column_encoding"] = {"s": ds.ENCODINGS[how]}
    sink = io.BytesIO()
    pq.write_table(ds.table(rows), sink, compression="LZ4" if lz4 else "NONE", data_page_version=version, row_group_size=rg,
                   store_schema=False, **kwargs)
    return sink.getvalue()


@functools.lru_cache(maxsize=None)
def str_file_of(name: str) -> bytes:
    return _str_write(name, True)


@functools.lru_cache(maxsize=None)
def str_twin_of(name: str) -> bytes:
    """The same pages uncompressed."""
    return _str_write(name, False)


def str_table(name: str) -> pa.Table:
    return ds.table(STR_CASES[name][0])


def str_schema() -> dp.Schema:
    s = ps.schema()
    for c in s.columns:
        c.compression = "LZ4_RAW"
    return s


# ---- LZ4 blocks from sequence plans ------------------------------------------------------------------------------
def _ext(n: int) -> bytes:
    return b"\xff" * (n // 255) + bytes([n % 255])


def encode(plan) -> bytes:
    """The block of a plan: per sequence the token, the literal length extension, the literals, the offset and the match
    length extension (the last sequence has no match)."""
    out = bytearray()
    for lits, m in plan:
        ll = len(lits)
        ml = m[1] - 4 if m else 0
        out.append((min(ll, 15) << 4) | (min(ml, 15) if m else 0))
        if ll >= 15:
            out += _ext(ll - 15)
        out += lits
        if m:
            out += struct.pack("<H", m[0])
            if ml >= 15:
                out += _ext(ml - 15)
    return bytes(out)


def execute(plan) -> bytes:
    """What a plan inflates to: a match repeats the `offset` bytes before it until it has `length` bytes."""
    out = bytearray()
    for lits, m in plan:
        out += lits
        if m:
            off, n = m
            pat = bytes(out[len(out) - off:])
            out += (pat * (n // off + 1))[:n]
    return bytes(out)


def _lits(seed: int, n: int) -> bytes:
    return np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8).tobytes()


def _tail(plan, seed: int):
    """Ends a plan with a literal-only sequence of >= 16 bytes that pads its output to a multiple of 8 bytes (the
    end-of-block rules: no match starts in the last 12 bytes nor ends in the last 5)."""
    n = len(execute(plan))
    return plan + [(_lits(seed, 16 + (-(n + 16)) % 8), None)]


def _valid_plans():
    head = _lits(2, 70000)  # room for offsets up to 65 535
    plans = {}
    for ll in (0, 14, 15, 270, 600):
        plans[f"literals_{ll}"] = [(_lits(3, 8), (8, 4)), (_lits(4 + ll, ll), (8, 4))]
    for ml in (4, 18, 19, 274):
        plans[f"match_{ml}"] = [(_lits(5, 8), (8, ml))]
    plans["match_1MiB_offset_1"] = [(_lits(6, 1), (1, 1 << 20))]
    for off in (1, 2, 3, 7, 8, 15, 16, 31, 32, 33, 4096, 65535):
        plans[f"offset_{off}"] = [(head, (off, 100)), (_lits(7, 3), (off, 4 * off + 5))]
    # a match copying what an earlier match wrote, and one reaching back into it from further on
    plans["match_of_match"] = [(_lits(8, 5), (5, 40)), (b"", (20, 60)), (_lits(9, 2), (77, 90))]
    plans["many_short_sequences"] = [(_lits(10, 16), (16, 4))] + [(_lits(11 + i, i % 5), (1 + (i * 7) % 16, 4 + i % 9)) for i in range(300)]
    out = {name: _tail(plan, 100 + i) for i, (name, plan) in enumerate(plans.items())}
    out["literal_only"] = [(_lits(12, 1000), None)]
    return out


@functools.lru_cache(maxsize=None)
def valid_blocks() -> List[Tuple[str, bytes, bytes]]:
    """(name, block, output) of the hand-assembled blocks, each checked with pyarrow's decoder, the empty block 0x00
    among them; and real blocks of pyarrow's compressor."""
    out = [(name, encode(plan), execute(plan)) for name, plan in _valid_plans().items()]
    out.append(("empty_0x00", b"\x00", b""))
    for name, data in (("pyarrow_runs", np.repeat(np.arange(300, dtype="<i8"), 37).tobytes()),
                       ("pyarrow_random", _lits(13, 4096)), ("pyarrow_timestamps", np.arange(10**12, 10**12 + 8000 * 15, 15, dtype="<i8").tobytes())):
        out.append((name, LZ4.compress(data, asbytes=True), data))
    for name, block, data in out:
        assert LZ4.decompress(block, decompressed_size=len(data), asbytes=True) == data, name
    return out


def pyarrow_accepts(block: bytes, size: int) -> bool:
    try:
        LZ4.decompress(block, decompressed_size=size, asbytes=True)
        return True
    except (OSError, pa.ArrowException):
        return False


# ---- malformed blocks: (name, block, size the header states, the engine's message) -------------------------------
def malformed():
    good = [(_lits(20, 40), (8, 30))]
    tail = [(_lits(21, 16), None)]
    blk = encode(good + tail)
    n = len(execute(good + tail))
    lit15 = encode([(_lits(22, 20), None)])
    p = "LZ4_RAW block: "
    return [
        ("offset_0", encode([(_lits(20, 40), (0, 30))] + tail), n, p + "match offset 0"),
        ("offset_past_output", encode([(_lits(20, 40), (41, 30))] + tail), n, p + "match offset reaches before the start of the output"),
        ("truncated_literals", encode([(_lits(23, 12), None)])[:-3], 12, p + "literal run runs past the block"),
        ("truncated_literal_extension", lit15[:1], 20, p + "literal length extension runs past the block"),
        ("truncated_match_extension", encode([(_lits(20, 40), (8, 2000))])[:44] + b"\xff" * 10, 4000,
         p + "match length extension runs past the block"),
        ("output_longer", blk, n - 8, p + "output longer than the header says"),
        ("output_shorter", blk, n + 8, p + "output shorter than the header says"),
        ("trailing_bytes", blk + b"\x00", n, p + "bytes behind the last sequence"),
        ("ends_with_a_match", encode(good) + b"\x00", len(execute(good)), p + "a match starts in the last 12 bytes of the output or the last 8 of the block"),
        ("match_in_last_5_bytes", encode(good + [(_lits(21, 4), None)]), n - 12, p + "a match ends in the last 5 bytes of the output"),
        ("empty_block", b"", 8, p + "empty (a block holds at least one token)"),
    ]


# pyarrow's decoder (liblz4's LZ4_decompress_safe into a buffer of the stated size) takes these too: it does not check
# that the block fills the buffer, and liblz4 copies a match of offset 0 instead of refusing it
PYARROW_TAKES = {"offset_0", "output_shorter"}


# ---- a page-level writer -----------------------------------------------------------------------------------------
PT_INT64 = 2
ENC_PLAIN, ENC_RLE, ENC_DBP, ENC_RLE_DICTIONARY = 0, 3, 5, 8
PAGE_DATA, PAGE_DICT, PAGE_DATA_V2 = 0, 2, 3


def _page(kind: str, n: int, enc: int, raw: bytes, block: Optional[bytes], raw_len: Optional[int] = None) -> bytes:
    """One page of a REQUIRED column: "v1" (the payload one block), "v2" (the values region one block) or "v2raw"
    (stored as it is, is_compressed false).  `block` None: pyarrow's compressor; `raw_len`: the inflated size the
    header states (default: the values' bytes)."""
    payload = raw if kind == "v2raw" else (LZ4.compress(raw, asbytes=True) if block is None else block)
    raw_len = len(raw) if raw_len is None else raw_len
    h = _Struct().i32(1, PAGE_DATA_V2 if kind.startswith("v2") else PAGE_DATA).i32(2, raw_len).i32(3, len(payload))
    if kind == "v1":
        h.struct(5, _Struct().i32(1, n).i32(2, enc).i32(3, ENC_RLE).i32(4, ENC_RLE))
    else:
        h.struct(8, _Struct().i32(1, n).i32(2, 0).i32(3, n).i32(4, enc).i32(5, 0).i32(6, 0).bool(7, kind == "v2"))
    return h.done() + payload


def assemble(pages, dictionary: Optional[List[int]] = None, codec: int = CODEC_LZ4_RAW, check: bool = True,
             encodings: Optional[List[int]] = None) -> bytes:
    """One row group: `value` (REQUIRED INT64, codec `codec`) from `pages`, a list of (kind, values, block or None[,
    stated inflated size]),
    behind a compressed dictionary page of `dictionary` when given (the pages then hold indices into it); `timestamp`
    (REQUIRED INT64, uncompressed PLAIN) 0 .. n-1.  `encodings`: per page ENC_PLAIN or ENC_DBP (tests/delta_int64.py's
    dbp64), PLAIN when not given.  With `check`, pyarrow must read `value` as the pages' values."""
    out = bytearray(b"PAR1")
    n = sum(len(p[1]) for p in pages)
    start = data_off = len(out)
    if dictionary is not None:
        d = np.asarray(dictionary, dtype="<i8").tobytes()
        blk = LZ4.compress(d, asbytes=True)
        out += _Struct().i32(1, PAGE_DICT).i32(2, len(d)).i32(3, len(blk)).struct(7, _Struct().i32(1, len(dictionary)).i32(2, ENC_PLAIN)).done() + blk
        data_off = len(out)
    expect = []
    encodings = encodings or [ENC_PLAIN] * len(pages)
    for (kind, values, block, *raw_len), value_enc in zip(pages, encodings):
        if dictionary is not None:
            idx = [dictionary.index(v) for v in values]
            w = max(1, max(idx).bit_length())
            raw, enc = bytes([w]) + encode_hybrid([bp(idx)], w), ENC_RLE_DICTIONARY
        elif value_enc == ENC_DBP:
            raw, enc = di.dbp64(values), ENC_DBP
        else:
            raw, enc = np.asarray(values, dtype="<i8").tobytes(), ENC_PLAIN
        pg = _page(kind, len(values), enc, raw, block, *raw_len)
        out += pg
        expect += [int(v) for v in values]
    v_size = len(out) - start
    encs = sorted({ENC_PLAIN, ENC_RLE} | set(encodings) | ({ENC_RLE_DICTIONARY} if dictionary is not None else set()))
    md = (_Struct().i32(1, PT_INT64).list(2, 5, [_zigzag(e) for e in encs]).list(3, 8, [_uleb(5) + b"value"]).i32(4, codec)
          .i64(5, n).i64(6, v_size).i64(7, v_size).i64(9, data_off))
    if dictionary is not None:
        md.i64(11, start)
    chunks = [_Struct().i64(2, start).struct(3, md).done()]
    t_start = len(out)
    t = np.arange(n, dtype="<i8").tobytes()
    out += _Struct().i32(1, PAGE_DATA).i32(2, len(t)).i32(3, len(t)).struct(5, _Struct().i32(1, n).i32(2, ENC_PLAIN).i32(3, ENC_RLE).i32(4, ENC_RLE)).done() + t
    t_size = len(out) - t_start
    md = (_Struct().i32(1, PT_INT64).list(2, 5, [_zigzag(ENC_PLAIN), _zigzag(ENC_RLE)]).list(3, 8, [_uleb(9) + b"timestamp"])
          .i32(4, 0).i64(5, n).i64(6, t_size).i64(7, t_size).i64(9, t_start))
    chunks.append(_Struct().i64(2, t_start).struct(3, md).done())
    rgs = [_Struct().list(1, 12, chunks).i64(2, v_size + t_size).i64(3, n).done()]
    schema_els = [_Struct().binary(4, b"schema").i32(5, 2).done(),
                  _Struct().i32(1, PT_INT64).i32(3, 0).binary(4, b"value").done(),
                  _Struct().i32(1, PT_INT64).i32(3, 0).binary(4, b"timestamp").done()]
    kv = [_Struct().binary(1, b"dynamic_columns").binary(2, b"").done()]
    footer = (_Struct().i32(1, 1).list(2, 12, schema_els).i64(3, n).list(4, 12, rgs).list(5, 12, kv)
              .binary(6, b"frostgpu tests (lz4_pages.py)").done())
    out += footer + struct.pack("<I", len(footer)) + b"PAR1"
    buf = bytes(out)
    if check:
        t = pq.read_table(io.BytesIO(buf))
        assert t.column("value").to_pylist() == expect, "pyarrow disagrees with the pages"
        assert t.column("timestamp").to_pylist() == list(range(n))
    return buf


def _i64(data: bytes) -> List[int]:
    return [int(x) for x in np.frombuffer(data, dtype="<i8")]


@functools.lru_cache(maxsize=None)
def hand_layouts():
    """(name, file, expected `value`, pages the device inflates) of the page-level layouts: every hand-assembled block
    with a non-empty output as a v1 page and as a v2 page, a v2 page stored uncompressed, the empty block as an empty
    page, and a compressed dictionary page with its index pages."""
    out = []
    for kind in ("v1", "v2"):  # one file per block, the empty block as a page of its own behind it
        for name, blk, data in valid_blocks():
            if data:
                out.append((f"{name}_{kind}", [(kind, _i64(data), blk), (kind, [], b"\x00")], 1))
    v = _i64(_lits(30, 800 * 8))
    out.append(("v2_stored_uncompressed", [("v2", v[:300], None), ("v2raw", v[300:500], None), ("v1", v[500:], None)], 2))
    out.append(("v2_empty_values_0_bytes", [("v2", v[:10], None), ("v2", [], b""), ("v2", v[10:20], None)], 2))
    files = [(name, assemble(pages), [x for p in pages for x in p[1]], dev) for name, pages, dev in out]
    d = [5, -3, ne.I64_MAX, 0]
    vals = [d[i % 4] for i in range(700)] + [d[(i * 7) % 3] for i in range(300)]
    pages = [("v1", vals[:400], None), ("v2", vals[400:], None)]
    files.append(("dictionary", assemble(pages, dictionary=d), vals, 0))
    return files


def corrupted_files():
    """(name, file, message): a malformed block as the v2 page of `value` behind a valid page."""
    v = _i64(_lits(31, 64))
    out = []
    for name, blk, size, message in malformed():
        if size < 8:
            continue
        vals = [0] * (size // 8)  # (the page header states `size`)
        out.append((name, assemble([("v2", v, None), ("v2", vals, blk, size)], check=False), message))
    return out


def codec_file(codec: int) -> bytes:
    """A chunk naming `codec` (its pages are LZ4_RAW, which does not matter: the codec is refused before any page)."""
    return assemble([("v1", list(range(10)), None)], codec=codec, check=False)


@functools.lru_cache(maxsize=None)
def mixed_fills():
    """(file, expected `value`): every way a page's values reach the dense value array, interleaved in one LZ4_RAW chunk.
    Its pages in order: a compressed PLAIN v1 page (the device inflates it), a DELTA_BINARY_PACKED v1 page (the host
    inflates it, the device decodes it from that buffer), a v2 PLAIN page stored uncompressed (copied as it is), a
    compressed PLAIN v2 page, and DELTA_BINARY_PACKED again."""
    a, c, d = _i64(_lits(40, 300 * 8)), _i64(_lits(41, 250 * 8)), _i64(_lits(42, 333 * 8))
    b = di._vals(43, 517)
    e = list(range(-10**15, -10**15 + 7 * 700, 7))
    pages = [("v1", a, None), ("v1", b, None), ("v2raw", c, None), ("v2", d, None), ("v1", e, None)]
    return assemble(pages, encodings=[ENC_PLAIN, ENC_DBP, ENC_PLAIN, ENC_PLAIN, ENC_DBP]), a + b + c + d + e
