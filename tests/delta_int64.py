"""Parquet parts whose int64 columns `timestamp` and `value` are written as DELTA_BINARY_PACKED pages, each with a PLAIN
twin holding the same rows.

- Layouts written by pyarrow through `dp.write_part` (`ColumnDefinition.delta_binary_packed`): sorted timestamps with
  step 1 (width-0 miniblocks), numeric_edges' INT_CHUNKS sorted and unsorted (frame-of-reference widths 8 .. 64 and
  both ends of int64), numeric_edges' wrap_part (full-range values: deltas wrap, miniblocks 64 bits wide), an OPTIONAL
  `value` with ~5 % NULLs, an all-NULL page and an all-NULL row group, small pages with row groups of 4 096 + 7 rows,
  data page v1 and v2, and numeric_edges' int_key_part (`value` as a group key).
- A small page-level writer for what pyarrow does not write: PLAIN and DELTA_BINARY_PACKED pages in one chunk, pages of
  0 and 1 values, other block and miniblock sizes, unused miniblocks with widths above 64, bytes behind a stream, one
  corrupted page per validation rule, DOUBLE with encoding 5 and a dictionary page followed by DELTA_BINARY_PACKED
  pages."""
import dataclasses
import functools
import io
import struct
from typing import Callable, Dict, List, Optional

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq

from frostdb_b200 import dynparquet as dp
from tests import numeric_edges as ne
from tests.delta_strings import _pack, _uleb, _zigzag
from tests.hybrid_pages import _Struct, bp, encode_hybrid

CK_PLAIN64 = 1
DBP = "DELTA_BINARY_PACKED"
I64_MIN, I64_MAX = ne.I64_MIN, ne.I64_MAX


def schema(cols: Dict[str, object], *, delta: bool, nullable_value: bool = False) -> dp.Schema:
    """numeric_edges' schema of `cols`, with `timestamp` and `value` DELTA_BINARY_PACKED when `delta`."""
    s = dp.SampleDefinitionWithFloat() if "floatvalue" in cols else dp.SampleDefinition()
    for c in s.columns:
        if c.name in ("timestamp", "value"):
            c.delta_binary_packed = delta
        if c.name == "value":
            c.nullable = nullable_value
    return s


def _nullable(seed: int, rg: int) -> Dict[str, object]:
    """Sorted INT_CHUNKS rows whose `value` is NULL in ~5 % of the rows, in rows [1 024, 3 072) of row group 0 (a whole
    write batch: an all-NULL page) and in all of row group 2."""
    cols = ne.int_part(ne.INT_CHUNKS[:4], seed, sort=True, rg=rg)
    n = len(cols["timestamp"])
    rng = np.random.default_rng(seed + 9)
    nulls = rng.random(n) < 0.05
    nulls[1024:3072] = True
    nulls[2 * rg:3 * rg] = True
    cols["value"] = pa.array(cols["value"], mask=nulls)
    return cols


@dataclasses.dataclass(frozen=True)
class Layout:
    name: str
    make: Callable[[], Dict[str, object]]
    sort: bool
    rg: int = ne.RG
    version: str = "2.0"
    data_page_size: Optional[int] = None
    nullable: bool = False


LAYOUTS = [
    Layout("sorted", lambda: ne.int_part(ne.INT_CHUNKS, 101, sort=True), True),
    Layout("unsorted", lambda: ne.int_part(ne.INT_CHUNKS, 102, sort=False), False),
    Layout("wrap", lambda: ne.wrap_part(6 * ne.RG, 103), False),
    Layout("nullable", lambda: _nullable(104, ne.RG), True, data_page_size=2048, nullable=True),
    Layout("page_edges", lambda: ne.int_part(ne.INT_CHUNKS, 105, sort=True, rg=ne.RG + 7), True, rg=ne.RG + 7, data_page_size=512),
    Layout("page_edges_v1", lambda: ne.int_part(ne.INT_CHUNKS[:3], 106, sort=False, rg=ne.RG + 7), False, rg=ne.RG + 7,
           version="1.0", data_page_size=700),
    Layout("sorted_v1", lambda: ne.int_part(ne.INT_CHUNKS, 107, sort=True), True, version="1.0"),
    Layout("int_key_sorted", lambda: ne.int_key_part(108, sort=True), True),
    Layout("int_key_unsorted", lambda: ne.int_key_part(109, sort=False), False),
]
LAYOUT_BY_NAME = {l.name: l for l in LAYOUTS}
NAMES = [l.name for l in LAYOUTS]


@functools.lru_cache(maxsize=None)
def columns(name: str) -> Dict[str, object]:
    """The layout's columns, without numeric_edges' `floatvalue` (its NaNs have no JSON form in a description)."""
    cols = LAYOUT_BY_NAME[name].make()
    cols.pop("floatvalue", None)
    return cols


def _write(name: str, delta: bool) -> bytes:
    l = LAYOUT_BY_NAME[name]
    cols = columns(name)
    kwargs = {} if l.data_page_size is None else {"data_page_size": l.data_page_size}
    return dp.write_part(schema(cols, delta=delta, nullable_value=l.nullable), cols, sort=False, row_group_size=l.rg,
                         data_page_version=l.version, **kwargs)


@functools.lru_cache(maxsize=None)
def file_of(name: str) -> bytes:
    """The layout with `timestamp` and `value` DELTA_BINARY_PACKED."""
    return _write(name, True)


@functools.lru_cache(maxsize=None)
def twin_of(name: str) -> bytes:
    """The same rows with `timestamp` and `value` PLAIN."""
    return _write(name, False)


def encodings(buf: bytes, column: str) -> List[set]:
    """Per row group, the value encodings the footer lists for `column`."""
    md = pq.ParquetFile(io.BytesIO(buf)).metadata
    names = [md.schema.column(i).path for i in range(md.num_columns)]
    j = names.index(column)
    return [set(md.row_group(g).column(j).encodings) - {"RLE", "BIT_PACKED"} for g in range(md.num_row_groups)]


def row_group_slices(buf: bytes):
    md = pq.ParquetFile(io.BytesIO(buf)).metadata
    out, b = [], 0
    for g in range(md.num_row_groups):
        n = md.row_group(g).num_rows
        out.append((b, b + n))
        b += n
    return out


def record_of(name: str) -> pa.RecordBatch:
    """The layout's rows as an Arrow record (dictionary labels as strings)."""
    t = dp.read_part(twin_of(name)).combine_chunks()
    cols = []
    for n in t.schema.names:
        c = t.column(n).chunk(0)
        if pa.types.is_dictionary(c.type):
            c = c.cast(pa.string())
        if pa.types.is_string(c.type):
            c = c.cast(pa.binary())
        cols.append(c)
    return pa.RecordBatch.from_arrays(cols, names=t.schema.names)


# ---- a page-level writer ----------------------------------------------------------------------------------------
PT_INT64, PT_DOUBLE = 2, 5
ENC_PLAIN, ENC_RLE, ENC_DBP, ENC_RLE_DICTIONARY = 0, 3, 5, 8
PAGE_DATA, PAGE_DICT = 0, 2
_M64 = (1 << 64) - 1


def _s64(x: int) -> int:
    x &= _M64
    return x - (1 << 64) if x >> 63 else x


def dbp64(values, block: int = 128, n_mb: int = 4, count: Optional[int] = None, width: Optional[int] = None,
          unused_width: int = 0) -> bytes:
    """DELTA_BINARY_PACKED of int64 values, deltas modulo 2^64 as the format has them: header, then per block the
    zigzag min delta, the miniblock bit widths and the miniblocks holding values, each whole.  `count` overrides the
    header's total, `width` the first bit width, `unused_width` the widths of the last block's unused miniblocks."""
    vals = [int(v) for v in values]
    out = _uleb(block) + _uleb(n_mb) + _uleb(len(vals) if count is None else count) + _zigzag(vals[0] if vals else 0)
    per = block // n_mb
    deltas = [_s64(vals[i] - vals[i - 1]) for i in range(1, len(vals))]
    for b in range(0, len(deltas), block):
        blk = deltas[b:b + block]
        mn = min(blk)
        rel = [(d - mn) & _M64 for d in blk]
        used = (len(rel) + per - 1) // per
        ws = [max(rel[m * per:(m + 1) * per]).bit_length() for m in range(used)] + [unused_width] * (n_mb - used)
        if width is not None and b == 0:
            ws[0] = width
        out += _zigzag(mn) + bytes(ws)
        for m in range(used):
            mb = rel[m * per:(m + 1) * per]
            out += _pack(mb + [0] * (per - len(mb)), min(ws[m], 64))
    return out


def _header(ptype: int, payload_len: int, sub_fid: int, sub) -> bytes:
    return _Struct().i32(1, ptype).i32(2, payload_len).i32(3, payload_len).struct(sub_fid, sub).done()


def _data_page(enc: int, n: int, payload: bytes) -> bytes:
    return _header(PAGE_DATA, len(payload), 5, _Struct().i32(1, n).i32(2, enc).i32(3, ENC_RLE).i32(4, ENC_RLE)) + payload


def assemble(pages, phys: int = PT_INT64, dictionary: Optional[List[int]] = None, check: bool = True) -> bytes:
    """One row group: `value` (REQUIRED INT64, or DOUBLE) from `pages`, a list of (encoding, values, payload or None
    for the encoding's own), behind a dictionary page of `dictionary` when given; `timestamp` (REQUIRED INT64, PLAIN)
    0 .. n-1.  With `check`, pyarrow must read `value` as the pages' values."""
    out = bytearray(b"PAR1")
    n = sum(len(v) for _, v, _ in pages)
    start = len(out)
    data_off = start
    if dictionary is not None:
        d = np.asarray(dictionary, dtype="<i8").tobytes()
        out += _header(PAGE_DICT, len(d), 7, _Struct().i32(1, len(dictionary)).i32(2, ENC_PLAIN)) + d
        data_off = len(out)
    expect = []
    for enc, values, payload in pages:
        if payload is None:
            if enc == ENC_RLE_DICTIONARY:
                idx = [dictionary.index(v) for v in values]
                w = max(1, max(idx).bit_length())
                payload = bytes([w]) + encode_hybrid([bp(idx)], w)
            elif enc == ENC_PLAIN:
                payload = np.asarray(values, dtype="<i8").tobytes()
            else:
                payload = dbp64(values)
        out += _data_page(enc, len(values), payload)
        expect += [int(v) for v in values]
    v_size = len(out) - start
    encs = sorted({e for e, _, _ in pages} | {ENC_RLE} | ({ENC_PLAIN} if dictionary is not None else set()))
    md = (_Struct().i32(1, phys).list(2, 5, [_zigzag(e) for e in encs]).list(3, 8, [_uleb(5) + b"value"]).i32(4, 0)
          .i64(5, n).i64(6, v_size).i64(7, v_size).i64(9, data_off))
    if dictionary is not None:
        md.i64(11, start)
    chunks = [_Struct().i64(2, start).struct(3, md).done()]
    t_start = len(out)
    out += _data_page(ENC_PLAIN, n, np.arange(n, dtype="<i8").tobytes())
    t_size = len(out) - t_start
    md = (_Struct().i32(1, PT_INT64).list(2, 5, [_zigzag(ENC_PLAIN), _zigzag(ENC_RLE)]).list(3, 8, [_uleb(9) + b"timestamp"])
          .i32(4, 0).i64(5, n).i64(6, t_size).i64(7, t_size).i64(9, t_start))
    chunks.append(_Struct().i64(2, t_start).struct(3, md).done())
    rgs = [_Struct().list(1, 12, chunks).i64(2, v_size + t_size).i64(3, n).done()]
    schema_els = [_Struct().binary(4, b"schema").i32(5, 2).done(),
                  _Struct().i32(1, phys).i32(3, 0).binary(4, b"value").done(),
                  _Struct().i32(1, PT_INT64).i32(3, 0).binary(4, b"timestamp").done()]
    kv = [_Struct().binary(1, b"dynamic_columns").binary(2, b"").done()]
    footer = (_Struct().i32(1, 1).list(2, 12, schema_els).i64(3, n).list(4, 12, rgs).list(5, 12, kv)
              .binary(6, b"frostgpu tests (delta_int64.py)").done())
    out += footer + struct.pack("<I", len(footer)) + b"PAR1"
    buf = bytes(out)
    if check:
        t = pq.read_table(io.BytesIO(buf))
        assert t.column("value").to_pylist() == expect, "pyarrow disagrees with the pages"
        assert t.column("timestamp").to_pylist() == list(range(n))
    return buf


def _vals(seed: int, n: int, lo: int = I64_MIN, hi: int = I64_MAX) -> List[int]:
    rng = np.random.default_rng(seed)
    return [int(x) for x in rng.integers(lo, hi, n, dtype=np.int64, endpoint=True)]


def hand_layouts():
    """(name, file, expected `value`) of the valid hand-assembled layouts."""
    a, b, c = _vals(1, 300, -1000, 1000), _vals(2, 517), list(range(10**12, 10**12 + 3 * 700, 3))
    one, big = [I64_MIN], _vals(3, 1000)
    cases = [
        ("mixed_plain_and_delta", [(ENC_PLAIN, a[:100], None), (ENC_DBP, a[100:], None), (ENC_PLAIN, b[:17], None),
                                   (ENC_DBP, b[17:], None), (ENC_DBP, c, None)]),
        ("one_and_zero_values", [(ENC_DBP, one, None), (ENC_DBP, [], None), (ENC_DBP, [I64_MAX], None), (ENC_DBP, b[:2], None),
                                 (ENC_DBP, [], None), (ENC_DBP, b[2:35], None)]),
        ("block_256_8_miniblocks", [(ENC_DBP, big, dbp64(big, block=256, n_mb=8)), (ENC_DBP, a, dbp64(a, block=256, n_mb=8))]),
        ("block_128_2_miniblocks", [(ENC_DBP, big, dbp64(big, block=128, n_mb=2)), (ENC_DBP, c, dbp64(c, block=128, n_mb=2))]),
        ("block_1024_1_miniblock", [(ENC_DBP, big, dbp64(big, block=1024, n_mb=1))]),
        ("unused_widths_above_64", [(ENC_DBP, a[:150], dbp64(a[:150], unused_width=200)), (ENC_DBP, b, dbp64(b, unused_width=65))]),
        ("bytes_behind_stream", [(ENC_DBP, a, dbp64(a) + b"\xff" * 13), (ENC_DBP, one, dbp64(one) + b"\x07")]),
    ]
    out = []
    for name, pages in cases:
        check = name != "unused_widths_above_64"  # (pyarrow checks the widths of unused miniblocks too)
        out.append((name, assemble(pages, check=check), [int(v) for _, vs, _ in pages for v in vs]))
    return out


def corrupted():
    """(name, file, message) per validation rule: one DELTA_BINARY_PACKED page that breaks it, behind a valid PLAIN page."""
    v = _vals(4, 300, -5000, 5000)
    head = (ENC_PLAIN, [7, 8], None)
    f = lambda payload: assemble([head, (ENC_DBP, v, payload)], check=False)
    over = "int64 values: DELTA_BINARY_PACKED stream overruns its page"
    whole = dbp64(v)
    hdr = len(_uleb(128) + _uleb(4) + _uleb(len(v)) + _zigzag(v[0]))
    return [
        ("block_size", f(dbp64(v, block=64, n_mb=2)), "int64 values: DELTA_BINARY_PACKED block size is not a multiple of 128"),
        ("miniblock_size", f(dbp64(v, block=128, n_mb=8)), "int64 values: DELTA_BINARY_PACKED miniblock size is not a multiple of 32"),
        ("count", f(dbp64(v, count=len(v) + 1)), "int64 values: DELTA_BINARY_PACKED value count differs from the page's values"),
        ("bit_width", f(dbp64(v, width=65)), "int64 values: DELTA_BINARY_PACKED miniblock bit width > 64"),
        ("header_overrun", f(whole[:hdr - 1]), over),
        ("widths_overrun", f(whole[:hdr + 2]), over),
        ("miniblock_overrun", f(whole[:-1]), over),
    ]


def double_delta() -> bytes:
    """DOUBLE `value` whose page is DELTA_BINARY_PACKED (the format allows it for INT32 / INT64 only)."""
    return assemble([(ENC_DBP, [1, 2, 3], None)], phys=PT_DOUBLE, check=False)


def dictionary_then_delta() -> bytes:
    """A numeric dictionary chunk whose writer fell back to DELTA_BINARY_PACKED pages."""
    d = [5, -3, I64_MAX]
    return assemble([(ENC_RLE_DICTIONARY, [5, 5, -3, I64_MAX], None), (ENC_DBP, _vals(5, 200), None)], dictionary=d, check=False)
