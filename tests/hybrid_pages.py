"""A page-level Parquet writer for tests, and the layout zoo of RLE / bit-packed hybrid streams built with it.

pyarrow writes a narrow subset of what the Parquet format allows for dictionary indices and definition levels: the
narrowest bit width (at least 1), one width per chunk, literal runs of at most 63 groups (one-byte run headers) and a
padded last group.  parquet-go, which writes FrostDB's parts, is not bound to that subset.  This module assembles
column chunks page by page from explicit run scripts, so every shape of the hybrid stream the decoder accepts can be
put in front of it:

- a script is a list of runs, `("rle", n, v)` or `("bp", values, trim)`; a bit-packed run holds ceil(len / 8) groups,
  and only the last run of a stream may hold a count that is not a multiple of 8 (its last group is padded with zeros,
  or, with `trim`, cut to the bytes its values need);
- a page has a row count, a bit width, the index script, for OPTIONAL columns a definition-level script, and a
  version (v1: levels behind a 4-byte length; v2: `definition_levels_byte_length` and `num_nulls`).

Files are uncompressed, with the columns of `dp.SampleDefinition()` (plus the INT64 dictionary column `dictvalue`)
and the `dynamic_columns` key-value metadata `dp.write_part` writes.  `decode_hybrid` is a plain decoder of the
hybrid stream; `write_file` decodes every page it wrote with it and asserts that the result, the values the scripts
stand for, and `pyarrow.parquet.read_table` agree on every column.  After that pyarrow's read is the reference.

`LAYOUTS` names every layout once; the host and GPU tests both take their files from it."""
from __future__ import annotations

import dataclasses
import functools
import io
import struct
from typing import Dict, List, Optional, Sequence

import numpy as np

from tests.bloom_file import Struct, _uvar, _zz

PT_INT64, PT_BYTE_ARRAY = 2, 6
ENC_PLAIN, ENC_RLE, ENC_RLE_DICTIONARY = 0, 3, 8
PAGE_DATA, PAGE_DICT, PAGE_DATA_V2 = 0, 2, 3
REQUIRED, OPTIONAL = 0, 1
CONVERTED_UTF8 = 0


class _Struct(Struct):
    def bool(self, fid, v: bool):
        self._hdr(fid, 1 if v else 2)
        return self


# ---- the hybrid stream -----------------------------------------------------------------------------------------
def rle(n: int, v: int):
    return ("rle", n, v)


def bp(values, trim: bool = False):
    return ("bp", [int(x) for x in values], trim)


def _pack(values: Sequence[int], w: int) -> bytes:
    acc = 0
    for i, v in enumerate(values):
        assert 0 <= v < (1 << w) or (w == 0 and v == 0), (v, w)
        acc |= v << (i * w)
    return acc.to_bytes((len(values) * w + 7) // 8, "little")


def encode_hybrid(script, w: int) -> bytes:
    out = bytearray()
    for i, run in enumerate(script):
        last = i == len(script) - 1
        if run[0] == "rle":
            _, n, v = run
            assert n > 0 and 0 <= v < max(1 << w, 1)
            out += _uvar(n << 1) + v.to_bytes((w + 7) // 8, "little")
        else:
            _, values, trim = run
            assert values and (last or len(values) % 8 == 0), "only the last run of a stream may end inside a group"
            assert not trim or last, "only the last group of a stream can be trimmed"
            groups = (len(values) + 7) // 8
            payload = _pack(values + [0] * (groups * 8 - len(values)), w)
            if trim:
                payload = payload[:(len(values) * w + 7) // 8]
            out += _uvar((groups << 1) | 1) + payload
    return bytes(out)


def script_values(script) -> List[int]:
    out: List[int] = []
    for run in script:
        out += [run[2]] * run[1] if run[0] == "rle" else run[1]
    return out


def decode_hybrid(buf: bytes, w: int, count: int) -> List[int]:
    """`count` values of a hybrid stream.  A bit-packed run's last group may be cut short at the end of the stream."""
    out: List[int] = []
    p = 0
    while len(out) < count:
        h, shift = 0, 0
        while True:
            b = buf[p]
            p += 1
            h |= (b & 0x7f) << shift
            shift += 7
            if not b & 0x80:
                break
        if h & 1:
            nbytes = (h >> 1) * w
            chunk = int.from_bytes(buf[p:p + nbytes], "little")
            mask = (1 << w) - 1
            out += [(chunk >> (i * w)) & mask for i in range((h >> 1) * 8)]
            p += nbytes
        else:
            vb = (w + 7) // 8
            assert h >> 1 > 0, "zero-length RLE run"
            out += [int.from_bytes(buf[p:p + vb], "little")] * (h >> 1)
            p += vb
    return out[:count]


# ---- pages and files -------------------------------------------------------------------------------------------
@dataclasses.dataclass
class Page:
    n: int                          # rows
    w: int                          # bit width of the dictionary indices
    idx: list                       # index script over the page's non-NULL values
    defs: Optional[list] = None     # definition-level script (OPTIONAL columns)
    v2: bool = False


@dataclasses.dataclass
class Column:
    name: str
    kind: str                       # "str" (BYTE_ARRAY/UTF8 dictionary), "i64dict" (INT64 dictionary), "plain" (INT64 PLAIN)
    required: bool = True
    pages: Optional[List[List[Page]]] = None   # per row group (dictionary columns)
    dictionary: Optional[list] = None
    values: Optional[List[np.ndarray]] = None  # per row group ("plain")


def _page_header(ptype: int, payload_len: int, sub_fid: int, sub: Struct) -> bytes:
    return _Struct().i32(1, ptype).i32(2, payload_len).i32(3, payload_len).struct(sub_fid, sub).done()


def _dict_page(col: Column) -> bytes:
    if col.kind == "str":
        data = b"".join(struct.pack("<I", len(s.encode())) + s.encode() for s in col.dictionary)
    else:
        data = struct.pack(f"<{len(col.dictionary)}q", *col.dictionary)
    return _page_header(PAGE_DICT, len(data), 7, _Struct().i32(1, len(col.dictionary)).i32(2, ENC_PLAIN)) + data


def _data_page(col: Column, pg: Page) -> bytes:
    defs = encode_hybrid(pg.defs, 1) if not col.required else b""
    values = bytes([pg.w]) + encode_hybrid(pg.idx, pg.w)
    nn = pg.n if col.required else sum(script_values(pg.defs))
    assert len(script_values(pg.idx)) == nn and (col.required or len(script_values(pg.defs)) == pg.n)
    if pg.v2:
        payload = defs + values
        h = (_Struct().i32(1, pg.n).i32(2, pg.n - nn).i32(3, pg.n).i32(4, ENC_RLE_DICTIONARY).i32(5, len(defs)).i32(6, 0)
             .bool(7, False))
        return _page_header(PAGE_DATA_V2, len(payload), 8, h) + payload
    payload = (struct.pack("<I", len(defs)) + defs if not col.required else b"") + values
    h = _Struct().i32(1, pg.n).i32(2, ENC_RLE_DICTIONARY).i32(3, ENC_RLE).i32(4, ENC_RLE)
    return _page_header(PAGE_DATA, len(payload), 5, h) + payload


def _decode_pages(col: Column, pages: List[bytes], rg: List[Page]) -> list:
    """The chunk's values, read back from the page bytes with decode_hybrid (None for NULL)."""
    out = []
    for raw, pg in zip(pages, rg):
        payload = raw[len(raw) - (_payload_len(col, pg)):]
        if col.required:
            levels, rest = [1] * pg.n, payload
        elif pg.v2:
            dl = len(encode_hybrid(pg.defs, 1))
            levels, rest = decode_hybrid(payload[:dl], 1, pg.n), payload[dl:]
        else:
            dl = struct.unpack_from("<I", payload)[0]
            levels, rest = decode_hybrid(payload[4:4 + dl], 1, pg.n), payload[4 + dl:]
        assert rest[0] == pg.w
        idx = iter(decode_hybrid(rest[1:], pg.w, sum(levels)))
        out += [col.dictionary[next(idx)] if lv else None for lv in levels]
    return out


def _payload_len(col: Column, pg: Page) -> int:
    defs = 0 if col.required else len(encode_hybrid(pg.defs, 1)) + (0 if pg.v2 else 4)
    return defs + 1 + len(encode_hybrid(pg.idx, pg.w))


def write_file(columns: List[Column], rg_rows: List[int], *, dict_page_offset: bool = True) -> bytes:
    """One file, one row group per entry of `rg_rows`, columns in name order; checked against pyarrow's read."""
    import pyarrow.parquet as pq
    columns = sorted(columns, key=lambda c: c.name)
    out = bytearray(b"PAR1")
    rgs, expect = [], {c.name: [] for c in columns}
    for g, n_rows in enumerate(rg_rows):
        chunks, rg_bytes = [], 0
        for col in columns:
            start = len(out)
            if col.kind == "plain":
                vals = np.asarray(col.values[g], dtype=np.int64)
                assert len(vals) == n_rows
                payload = vals.astype("<i8").tobytes()
                out += _page_header(PAGE_DATA, len(payload), 5, _Struct().i32(1, n_rows).i32(2, ENC_PLAIN).i32(3, ENC_RLE).i32(4, ENC_RLE))
                out += payload
                expect[col.name] += vals.tolist()
                data_off, ptype = start, PT_INT64
                stats = _Struct().i64(3, 0).binary(5, struct.pack("<q", int(vals.max()))).binary(6, struct.pack("<q", int(vals.min())))
            else:
                rg = col.pages[g]
                assert sum(p.n for p in rg) == n_rows
                out += _dict_page(col)
                data_off = len(out)
                raw = [_data_page(col, pg) for pg in rg]
                for r in raw:
                    out += r
                got = _decode_pages(col, raw, rg)
                want = []
                for pg in rg:
                    idx = iter(script_values(pg.idx))
                    levels = [1] * pg.n if col.required else script_values(pg.defs)
                    want += [col.dictionary[next(idx)] if lv else None for lv in levels]
                assert got == want, f"{col.name}: the decoder disagrees with the scripts"
                expect[col.name] += want
                ptype, stats = (PT_BYTE_ARRAY if col.kind == "str" else PT_INT64), None
            size = len(out) - start
            rg_bytes += size
            md = (_Struct().i32(1, ptype).list(2, 5, [_zz(ENC_PLAIN), _zz(ENC_RLE), _zz(ENC_RLE_DICTIONARY)])
                  .list(3, 8, [_uvar(len(col.name)) + col.name.encode()]).i32(4, 0).i64(5, n_rows).i64(6, size).i64(7, size)
                  .i64(9, data_off if (col.kind == "plain" or dict_page_offset) else start))
            if col.kind != "plain" and dict_page_offset:
                md.i64(11, start)
            if stats is not None:
                md.struct(12, stats)
            chunks.append(_Struct().i64(2, start).struct(3, md).done())
        rgs.append(_Struct().list(1, 12, chunks).i64(2, rg_bytes).i64(3, n_rows).done())
    schema = [_Struct().binary(4, b"schema").i32(5, len(columns)).done()]
    for col in columns:
        s = _Struct().i32(1, PT_BYTE_ARRAY if col.kind == "str" else PT_INT64).i32(3, REQUIRED if col.required else OPTIONAL)
        s.binary(4, col.name.encode())
        if col.kind == "str":
            s.i32(6, CONVERTED_UTF8)
        schema.append(s.done())
    dyn = sorted(c.name.split(".", 1)[1] for c in columns if c.name.startswith("labels."))
    kv = [_Struct().binary(1, b"dynamic_columns").binary(2, ("labels:" + ",".join(dyn)).encode()).done()]
    footer = (_Struct().i32(1, 1).list(2, 12, schema).i64(3, sum(rg_rows)).list(4, 12, rgs).list(5, 12, kv)
              .binary(6, b"frostgpu tests (hybrid_pages.py)").done())
    out += footer + struct.pack("<I", len(footer)) + b"PAR1"
    buf = bytes(out)
    t = pq.read_table(io.BytesIO(buf))
    for col in columns:
        assert t.column(col.name).to_pylist() == expect[col.name], f"pyarrow disagrees on {col.name}"
    return buf


# ---- the layout zoo --------------------------------------------------------------------------------------------
@dataclasses.dataclass
class Layout:
    """The zoo column `labels.z` (and `dictvalue`, the same pages over an INT64 dictionary).

    sorted: the zoo column is run-length only with long runs, so aggregates keyed by it take the sorted-run kernel;
    otherwise it holds bit-packed runs and they take the tile kernel.  n_runs / n_row_runs: the value-stream directory
    and the row-space directory each row group must get.  error: the chunk must be refused with this message.
    repeats: dictionary entry i holds the value of entry repeats[i] (a dictionary page that repeats entries)."""
    name: str
    dict_size: int
    pages: List[List[Page]]
    required: bool = True
    sorted: bool = False
    n_runs: Optional[List[int]] = None
    n_row_runs: Optional[List[int]] = None
    error: Optional[str] = None
    dict_page_offset: bool = True
    repeats: Optional[List[int]] = None

    @property
    def rg_rows(self) -> List[int]:
        return [sum(p.n for p in rg) for rg in self.pages]

    def entry(self, i: int) -> int:
        return self.repeats[i] if self.repeats else i

    @property
    def z_dictionary(self) -> List[str]:
        return [f"z{self.entry(i):03d}" for i in range(self.dict_size)]

    @property
    def dictvalue_dictionary(self) -> List[int]:
        return [(j * 7919) % 1009 - 504 + j * (1 << 33) for j in map(self.entry, range(self.dict_size))]


def _rand(seed: int, hi: int, n: int) -> List[int]:
    return np.random.default_rng(seed).integers(0, hi, n).tolist()


def _bits(seed: int, n: int, p_null: float = 0.2) -> List[int]:
    return (np.random.default_rng(seed).random(n) >= p_null).astype(int).tolist()


def _nullable_bp_page(seed: int, n: int, w: int, hi: int, defs_head=(), idx_head=(), v2=False) -> Page:
    """A page whose definition levels end in a bit-packed run of random levels and whose indices end in a bit-packed
    run of random values."""
    head = sum(r[1] for r in defs_head)
    head_nn = sum(script_values(list(defs_head)))
    tail = _bits(seed, n - head)
    idx_head_n = sum(r[1] for r in idx_head)
    nn = head_nn + sum(tail)
    return Page(n, w, list(idx_head) + [bp(_rand(seed + 1, hi, nn - idx_head_n))], defs=list(defs_head) + [bp(tail)], v2=v2)


P = Page
LAYOUTS: List[Layout] = [
    # one-entry dictionary at bit width 0: RLE runs (merged within and across pages) ...
    Layout("width0_rle", 1, [[P(5003, 0, [rle(2000, 0), rle(3003, 0)])],
                             [P(1501, 0, [rle(1501, 0)]), P(1576, 0, [rle(1576, 0)], v2=True)]],
           sorted=True, n_runs=[1, 1]),
    # ... and bit-packed runs without payload (a width-0 bit-packed run is recorded as an RLE run of entry 0)
    Layout("width0_bitpacked", 1, [[P(5003, 0, [bp([0] * 5003)])],
                                   [P(777, 0, [bp([0] * 24), rle(753, 0)]), P(2300, 0, [bp([0] * 2300)], v2=True)]],
           sorted=True, n_runs=[1, 1]),
    # 5 entries at widths 3, 12, 24, 8 and 16 in one chunk, and 20: the LUT and dict64 are padded to 2^w entries per
    # chunk; RLE values of 3 bytes at widths 20 and 24
    Layout("over_wide", 5, [[P(4099, 3, [bp(_rand(1, 5, 4099))])],
                            [P(3001, 12, [bp(_rand(2, 5, 1504)), bp(_rand(3, 5, 1497))])],
                            [P(2053, 24, [bp(_rand(4, 5, 2053), trim=True)], v2=True), P(500, 24, [rle(500, 3)])],
                            [P(1001, 8, [bp(_rand(20, 5, 1001))]), P(999, 16, [bp(_rand(21, 5, 992)), rle(7, 4)], v2=True)],
                            [P(2001, 20, [rle(1000, 2), bp(_rand(22, 5, 1001), trim=True)])]],
           n_runs=[1, 2, 2, 3, 2]),
    # bit-packed indices wider than a 5-entry dictionary can need, beyond 24 bits: refused, not decoded
    Layout("refused_width25", 5, [[P(1000, 25, [bp(_rand(5, 5, 1000))])]], error="wider than the dictionary"),
    Layout("refused_width32", 5, [[P(1000, 32, [bp(_rand(6, 5, 1000))])]], error="wider than the dictionary"),
    # whole pages as single bit-packed runs (2-byte headers) at widths 3, 5, 7, the last group trimmed to 377, 626,
    # 1753 and 1254 bytes or padded; widths change from page to page inside one 128-row chunk
    Layout("bitpacked_trimmed", 100, [[P(1003, 3, [bp(_rand(7, 8, 1003), trim=True)]),
                                       P(1001, 5, [bp(_rand(8, 32, 1001), trim=True)], v2=True),
                                       P(2003, 7, [bp(_rand(9, 100, 2003), trim=True)])],
                                      [P(1003, 3, [bp(_rand(10, 8, 1003))]), P(2005, 5, [bp(_rand(11, 32, 2005), trim=True)])]],
           n_runs=[3, 2]),
    # run-length pages at widths 3, 7, 1 and 12, 9: one value's run continues across pages; an "aaaaabbb" spill
    Layout("page_widths", 100, [[P(1003, 3, [rle(700, 5), rle(303, 6)]),
                                 P(517, 7, [rle(211, 6), bp([6] * 6 + [70] * 2), rle(298, 70)], v2=True),
                                 P(1203, 1, [rle(600, 1), rle(603, 0)])],
                                [P(800, 12, [rle(800, 99)]), P(797, 9, [rle(400, 99), rle(397, 98)])]],
           sorted=True, n_runs=[5, 2]),
    # literal runs of 8 and 64 values are unpacked: a spill between RLE runs, a 64-value literal across two values,
    # literals equal to both neighbours (one directory run), and across a page boundary
    Layout("short_literals", 20, [[P(1681, 5, [rle(300, 0), bp([0] * 5 + [1] * 3), rle(301, 1), bp([1] * 10 + [2] * 54),
                                               rle(203, 2), bp([2] * 8), rle(400, 2), bp([3] * 64), rle(333, 3)])],
                                  [P(1000, 5, [rle(992, 4), bp([4] * 3 + [5] * 5)]),
                                   P(1100, 5, [bp([5] * 8), rle(1092, 5)], v2=True)]],
           sorted=True, n_runs=[4, 2]),
    # a 72-value literal stays one bit-packed run (a 64-value one between equal RLE runs still merges)
    Layout("literal_72", 300, [[P(2211, 9, [rle(500, 7), bp(_rand(12, 300, 72)), rle(500, 8), bp([8] * 64),
                                            bp(_rand(13, 300, 72)), rle(1003, 9)])]],
           n_runs=[5]),
    # RLE run headers of 1, 2 and 3 bytes (63, 64 and 2^14 values) ...
    Layout("rle_headers", 10, [[P(17512, 4, [rle(63, 0), rle(64, 1), rle(1 << 14, 2), rle(1001, 3)])]],
           sorted=True, n_runs=[4]),
    # ... and of 4 bytes (2^21 + 3 values: above the host decode's 65536-row limit, checked on the GPU)
    Layout("rle_4byte_header", 10, [[P((1 << 21) + 3 + 1290, 4, [rle((1 << 21) + 3, 4), rle(1290, 5)])]],
           sorted=True, n_runs=[2]),
    # OPTIONAL, run-length levels and indices (the row-space directory): NULL runs ending and starting on 128-row
    # boundaries, an all-NULL v2 page in the middle of a chunk, a value run continuing across it, v1 and v2 pages
    Layout("nullable_rle", 10, [[P(1280, 4, [rle(1024, 0)], defs=[rle(256, 0), rle(1024, 1)]),
                                 P(771, 4, [], defs=[rle(771, 0)], v2=True),
                                 P(2048, 4, [rle(500, 0), rle(1548, 1)], defs=[rle(2048, 1)])],
                                [P(1111, 4, [rle(1111, 2)], defs=[rle(1111, 1)], v2=True),
                                 P(2222, 4, [rle(300, 2), rle(700, 3)], defs=[rle(1000, 1), rle(1222, 0)])]],
           required=False, sorted=True, n_runs=[2, 2], n_row_runs=[5, 3]),
    # OPTIONAL, run-length, a dictionary page that repeats an entry: indices 0 and 2 stand for the same value, two
    # value runs that the row-space directory merges into one (global ids), also across a page boundary
    Layout("nullable_rle_repeated_entry", 3, [[P(1000, 2, [rle(400, 0), rle(344, 2)], defs=[rle(256, 0), rle(744, 1)]),
                                               P(1303, 2, [rle(103, 2), rle(200, 1)], defs=[rle(303, 1), rle(1000, 0)], v2=True)],
                                              [P(1501, 2, [rle(601, 2), rle(399, 0)], defs=[rle(1000, 1), rle(501, 0)])]],
           required=False, sorted=True, n_runs=[3, 2], n_row_runs=[4, 2], repeats=[0, 1, 0]),
    # OPTIONAL, bit-packed definition levels and indices, v1 and v2
    Layout("nullable_bitpacked", 50, [[_nullable_bp_page(14, 1500, 6, 50),
                                       _nullable_bp_page(16, 1501, 6, 50, defs_head=[rle(64, 0)], v2=True)],
                                      [_nullable_bp_page(18, 2049, 6, 50, defs_head=[rle(1000, 1)], idx_head=[rle(504, 3)])]],
           required=False, n_runs=[2, 2]),
    # the dictionary page found through data_page_offset, dictionary_page_offset unset
    Layout("dictionary_via_data_page_offset", 3, [[P(3000, 2, [rle(1000, 0), rle(1000, 1), rle(1000, 2)])],
                                                  [P(1777, 2, [rle(1777, 2)])]],
           sorted=True, n_runs=[3, 1], dict_page_offset=False),
]
LAYOUT_BY_NAME: Dict[str, Layout] = {l.name: l for l in LAYOUTS}
assert len(LAYOUT_BY_NAME) == len(LAYOUTS)


def _y_pages(layout: Layout, g: int, n: int) -> List[Page]:
    """The second key, labels.y (3 entries, width 2): runs of 1000 rows for sorted layouts, bit-packed otherwise."""
    if layout.sorted:
        return [Page(n, 2, [rle(min(1000, n - s), (s // 1000) % 3) for s in range(0, n, 1000)])]
    return [Page(n, 2, [bp(_rand(100 + g, 3, n))])]


def columns(layout: Layout) -> List[Column]:
    rows = layout.rg_rows
    rng = np.random.default_rng(1000 + len(layout.name))
    t0 = np.cumsum([0] + rows)
    return [
        Column("example_type", "str", pages=[[Page(n, 0, [rle(n, 0)])] for n in rows], dictionary=["cpu"]),
        Column("stacktrace", "str", pages=[[Page(n, 0, [bp([0] * n)])] for n in rows], dictionary=["s"]),
        Column("labels.y", "str", pages=[_y_pages(layout, g, n) for g, n in enumerate(rows)], dictionary=["y0", "y1", "y2"]),
        Column("labels.z", "str", required=layout.required, pages=layout.pages, dictionary=layout.z_dictionary),
        Column("dictvalue", "i64dict", required=layout.required, pages=layout.pages, dictionary=layout.dictvalue_dictionary),
        Column("timestamp", "plain", values=[np.arange(t0[g], t0[g + 1], dtype=np.int64) for g in range(len(rows))]),
        Column("value", "plain", values=[rng.integers(-(1 << 31), 1 << 31, n, dtype=np.int64) for n in rows]),
    ]


@functools.lru_cache(maxsize=None)
def file_of(name: str) -> bytes:
    layout = LAYOUT_BY_NAME[name]
    return write_file(columns(layout), layout.rg_rows, dict_page_offset=layout.dict_page_offset)


def read(name: str):
    """pyarrow's read of a zoo file: the reference."""
    import pyarrow.parquet as pq
    return pq.read_table(io.BytesIO(file_of(name)))


def schema():
    """dp.SampleDefinition() plus the nullable INT64 dictionary column `dictvalue`."""
    from frostdb_b200 import dynparquet as dp
    s = dp.SampleDefinition()
    s.columns.append(dp.ColumnDefinition("dictvalue", dp.TYPE_INT64, nullable=True))
    return s


# ---- the reference: numpy over pyarrow's read --------------------------------------------------------------------
class Reference:
    """Plans over one zoo file, evaluated with numpy on pyarrow's read.  A leaf never selects NULL except `== NULL`;
    a NULL `dictvalue` contributes 0 to Sum / Max (the engine's NULL slot); Count counts rows; results are exact."""

    def __init__(self, name: str):
        import pyarrow as pa
        t = read(name)
        self.n = t.num_rows
        self.str_cols, self.int_cols = {}, {}
        for c in t.column_names:
            a = t.column(c).combine_chunks()
            if pa.types.is_string(a.type):
                enc = a.dictionary_encode()
                self.str_cols[c] = (enc.indices.fill_null(-1).to_numpy(zero_copy_only=False).astype(np.int64),
                                    enc.dictionary.to_pylist())
            else:
                self.int_cols[c] = (a.fill_null(0).to_numpy(zero_copy_only=False).astype(np.int64),
                                    a.is_null().to_numpy(zero_copy_only=False))

    def mask(self, filt) -> np.ndarray:
        import re
        from frostdb_b200 import logicalplan as lp
        if filt is None:
            return np.ones(self.n, bool)
        if filt.Op == lp.OpAnd:
            return self.mask(filt.Left) & self.mask(filt.Right)
        if filt.Op == lp.OpOr:
            return self.mask(filt.Left) | self.mask(filt.Right)
        name, op, lit = filt.Left.Name(), filt.Op, filt.Right.Value
        if name in self.str_cols:
            codes, d = self.str_cols[name]
            valid = codes >= 0
            if lit is None:
                return {lp.OpEq: ~valid, lp.OpNotEq: valid}[op]
            if op in (lp.OpRegexMatch, lp.OpRegexNotMatch):
                hit = np.array([re.search(lit, x) is not None for x in d] + [False], bool)
                return valid & (hit[codes] if op == lp.OpRegexMatch else ~hit[codes])
            hit = np.array([x == lit for x in d] + [False], bool)
            return {lp.OpEq: valid & hit[codes], lp.OpNotEq: valid & ~hit[codes]}[op]
        x, null = self.int_cols[name]
        y = np.int64(lit)
        return ~null & {lp.OpEq: x == y, lp.OpNotEq: x != y, lp.OpLt: x < y, lp.OpLtEq: x <= y, lp.OpGt: x > y,
                        lp.OpGtEq: x >= y}[op]

    def aggregate(self, filt, keys: Sequence[str], aggs) -> dict:
        """{key tuple (str or None): tuple of aggregate values}."""
        from frostdb_b200 import logicalplan as lp
        sel = np.flatnonzero(self.mask(filt))
        if len(sel) == 0:
            return {}
        combined = np.zeros(len(sel), np.int64)
        for k in keys:
            combined = combined * (len(self.str_cols[k][1]) + 1) + self.str_cols[k][0][sel] + 1
        ucomb, gid = np.unique(combined, return_inverse=True)
        uniq = np.zeros((len(keys), len(ucomb)), np.int64)
        for i, k in reversed(list(enumerate(keys))):
            uniq[i] = ucomb % (len(self.str_cols[k][1]) + 1) - 1
            ucomb //= len(self.str_cols[k][1]) + 1
        gid = gid.reshape(-1)
        order = np.argsort(gid, kind="stable")
        starts = np.flatnonzero(np.r_[True, np.diff(gid[order]) != 0])
        out_cols = []
        for a in aggs:
            if a.Func == lp.AggFuncCount:
                out_cols.append(np.diff(np.r_[starts, len(sel)]).tolist())
                continue
            v = self.int_cols[a.Expr.Name()][0][sel][order]
            ufunc = {lp.AggFuncSum: np.add, lp.AggFuncMin: np.minimum, lp.AggFuncMax: np.maximum}[a.Func]
            out_cols.append(ufunc.reduceat(v, starts).tolist())
        out = {}
        for j in range(uniq.shape[1]):
            key = tuple(None if uniq[i, j] < 0 else self.str_cols[k][1][uniq[i, j]] for i, k in enumerate(keys))
            out[key] = tuple(c[j] for c in out_cols)
        return out

    def rows(self, filt, names: Sequence[str]) -> Dict[str, "pa.Array"]:
        """Filter-only plans: the selected rows in file order, one array per column."""
        import pyarrow as pa
        sel = np.flatnonzero(self.mask(filt))
        out = {}
        for n in names:
            if n in self.str_cols:
                codes, d = self.str_cols[n]
                c = codes[sel]
                out[n] = pa.DictionaryArray.from_arrays(pa.array(np.maximum(c, 0).astype(np.int32), mask=c < 0),
                                                        pa.array(d, pa.string())).dictionary_decode()
            else:
                x, null = self.int_cols[n]
                out[n] = pa.array(x[sel], mask=null[sel])
        return out


def zoo_literal(layout: Layout) -> str:
    return layout.z_dictionary[1 % layout.dict_size]


def zoo_filters(layout: Layout):
    """Leaves on labels.z and timestamp ranges: what the take kernels evaluate (dictionary leaves on flat codes)."""
    from frostdb_b200 import logicalplan as lp
    z, n, lit, ts = lp.Col("labels.z"), sum(layout.rg_rows), zoo_literal(layout), lp.Col("timestamp")
    return [lp.And(ts.GtEq(lp.Literal(n // 3)), ts.Lt(lp.Literal(2 * n // 3))),
            z.Eq(lp.Literal(lit)), z.NotEq(lp.Literal(lit)), z.Eq(lp.Literal(None)), z.NotEq(lp.Literal(None)),
            z.RegexMatch("z00[13579]"), lp.And(z.NotEq(lp.Literal(lit)), ts.GtEq(lp.Literal(1)))]


def plans(layout: Layout):
    """(filter, keys, aggregates) of the aggregate plans run on every zoo file."""
    from frostdb_b200 import logicalplan as lp
    filters = [None] + zoo_filters(layout) + [lp.Col("dictvalue").Gt(lp.Literal(0))]
    value_aggs = [lp.Sum(lp.Col("value")), lp.Count(lp.Col("value")), lp.Min(lp.Col("value")), lp.Max(lp.Col("value"))]
    dict_aggs = [lp.Sum(lp.Col("dictvalue")), lp.Max(lp.Col("dictvalue"))]
    return [(f, keys, aggs) for f in filters for keys in (["labels.z"], ["labels.z", "labels.y"]) for aggs in (value_aggs, dict_aggs)]
