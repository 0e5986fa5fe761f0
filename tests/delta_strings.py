"""Parquet parts whose string column `s` is written as DELTA_LENGTH_BYTE_ARRAY (DLBA) or DELTA_BYTE_ARRAY (DBA) pages,
each with an RLE_DICTIONARY twin and a PLAIN twin holding the same rows.

- Every PLAIN layout of tests/plain_strings.py (its dictionary-fallback layouts aside) in both encodings, written by
  pyarrow with `use_dictionary=False, column_encoding=...`.
- DBA layouts whose front coding matters: sorted values with long shared prefixes (runs of 1 024 values inside one page
  start with a prefix on the run before), values equal to their predecessor (empty suffixes), a chain of 1 200 values
  each extending the previous one and then one with prefix 0, and pages of sorted values, so that a page's first value
  would share a prefix with the page before.
- A small page-level writer for what pyarrow cannot write: one chunk whose dictionary page and dictionary-index page are
  followed by DLBA, DBA and PLAIN pages, and DLBA / DBA pages that break one validation rule each.

Every layout has the columns `s`, `timestamp` (int64, unique), `value` (int64) and `fvalue` (double, nullable)."""
import dataclasses
import functools
import io
import struct
from typing import List, Optional

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq

from tests import plain_strings as ps
from tests.hybrid_pages import _Struct, bp, encode_hybrid

CK_DICT_STR = ps.CK_DICT_STR
ENCODINGS = {"dlba": "DELTA_LENGTH_BYTE_ARRAY", "dba": "DELTA_BYTE_ARRAY"}


@dataclasses.dataclass(frozen=True)
class Front:
    """A DBA layout: the rows of `s` come from `kind`."""
    name: str
    kind: str
    n_rows: int
    seed: int
    version: str = "2.0"
    nullable: bool = False
    null_p: float = 0.0
    data_page_size: Optional[int] = None
    write_batch_size: Optional[int] = None


FRONTS = [
    Front("sorted_prefixes", "sorted", 20000, 21, data_page_size=1 << 20),
    Front("repeated_values", "repeats", 6000, 22, version="1.0", nullable=True, null_p=0.1, data_page_size=4096),
    Front("long_chain", "chain", 1300, 23, data_page_size=1 << 22),
    Front("page_edges", "sorted", 4000, 24, nullable=True, null_p=0.05, data_page_size=512, write_batch_size=32),
]
FRONT_BY_NAME = {f.name: f for f in FRONTS}

PLAIN_NAMES = [l.name for l in ps.LAYOUTS if not l.fallback]
# (layout, encoding) of every file: the PLAIN layouts in both encodings, the front-coding layouts in DBA
CASES = [(n, e) for n in PLAIN_NAMES for e in ENCODINGS] + [(f.name, "dba") for f in FRONTS]
CASE_IDS = [f"{n}-{e}" for n, e in CASES]


def _front_strings(f: Front, rng) -> List[str]:
    if f.kind == "sorted":
        return sorted(f"/usr/lib/python3/site-packages/module_{i // 7:06d}/frame_{i % 7}_{int(rng.integers(0, 4))}"
                      for i in range(f.n_rows))
    if f.kind == "repeats":
        out = []
        while len(out) < f.n_rows:
            v = "shared/prefix/" + "".join(chr(c) for c in rng.integers(0x61, 0x7b, size=int(rng.integers(0, 12))))
            out += [v] * int(rng.integers(1, 6))
        return out[: f.n_rows]
    assert f.kind == "chain"
    letters = "".join(chr(0x61 + (k % 26)) for k in range(1200))
    chain = [letters[: i + 1] for i in range(1200)]
    return (chain + ["zz-no-prefix"] + [chain[int(i)] for i in rng.integers(0, 1200, size=f.n_rows - 1201)])[: f.n_rows]


@functools.lru_cache(maxsize=None)
def table(name: str) -> pa.Table:
    if name not in FRONT_BY_NAME:
        return ps.table(name)
    f = FRONT_BY_NAME[name]
    rng = np.random.default_rng(f.seed)
    s = _front_strings(f, rng)
    nulls = rng.random(f.n_rows) < f.null_p
    s = [None if n else v for v, n in zip(s, nulls)]
    fv = rng.normal(size=f.n_rows) * 100.0
    fields = [pa.field("fvalue", pa.float64(), nullable=True), pa.field("s", pa.string(), nullable=f.nullable),
              pa.field("timestamp", pa.int64(), nullable=False), pa.field("value", pa.int64(), nullable=False)]
    arrays = [pa.array(fv, mask=rng.random(f.n_rows) < 0.1), pa.array(s, type=pa.string()),
              pa.array(np.arange(f.n_rows, dtype=np.int64)), pa.array(rng.integers(-1000, 1000, size=f.n_rows))]
    return pa.Table.from_arrays(arrays, schema=pa.schema(fields)).replace_schema_metadata({"dynamic_columns": ""})


def _write(name: str, how: str) -> bytes:
    """how: "dlba" / "dba" (the layout), "dict" (RLE_DICTIONARY twin) or "plain" (PLAIN twin)."""
    if name in FRONT_BY_NAME:
        f = FRONT_BY_NAME[name]
        version, rg, page, batch = f.version, f.n_rows, f.data_page_size, f.write_batch_size
    else:
        l = ps.LAYOUT_BY_NAME[name]
        version, rg, page, batch = l.version, l.row_group_size or max(l.n_rows, 1), l.data_page_size, l.write_batch_size
    kwargs = {}
    if page is not None:
        kwargs["data_page_size"] = page
    if batch is not None:
        kwargs["write_batch_size"] = batch
    if how == "dict":
        kwargs["dictionary_pagesize_limit"] = 1 << 28
        kwargs["use_dictionary"] = ["s"]
    else:
        kwargs["use_dictionary"] = False
        if how in ENCODINGS:
            kwargs["column_encoding"] = {"s": ENCODINGS[how]}
    sink = io.BytesIO()
    pq.write_table(table(name), sink, compression="NONE", data_page_version=version, row_group_size=rg, store_schema=False, **kwargs)
    return sink.getvalue()


@functools.lru_cache(maxsize=None)
def file_of(name: str, enc: str) -> bytes:
    return _write(name, enc)


@functools.lru_cache(maxsize=None)
def twin_of(name: str) -> bytes:
    """The same rows with `s` RLE_DICTIONARY throughout."""
    return _write(name, "dict")


@functools.lru_cache(maxsize=None)
def plain_of(name: str) -> bytes:
    """The same rows with `s` PLAIN."""
    return _write(name, "plain")


def record_of(name: str) -> pa.RecordBatch:
    t = table(name).combine_chunks()
    cols = [t.column(n).chunk(0) if t.num_rows else pa.array([], t.schema.field(n).type) for n in t.schema.names]
    cols = [c.cast(pa.binary()) if n == "s" else c for n, c in zip(t.schema.names, cols)]
    return pa.RecordBatch.from_arrays(cols, names=t.schema.names)


s_encodings = ps.s_encodings
row_group_slices = ps.row_group_slices
first_occurrence = ps.first_occurrence
schema = ps.schema


# ---- a page-level writer ----------------------------------------------------------------------------------------
PT_INT64, PT_BYTE_ARRAY = 2, 6
ENC_PLAIN, ENC_RLE, ENC_DLBA, ENC_DBA, ENC_RLE_DICTIONARY = 0, 3, 6, 7, 8
PAGE_DATA, PAGE_DICT = 0, 2


def _uleb(n: int) -> bytes:
    assert n >= 0
    out = bytearray()
    while True:
        b, n = n & 0x7f, n >> 7
        out.append(b | (0x80 if n else 0))
        if not n:
            return bytes(out)


def _zigzag(n: int) -> bytes:
    return _uleb((n << 1) ^ (n >> 63) if n < 0 else n << 1)


def _pack(values, w: int) -> bytes:
    acc = 0
    for i, v in enumerate(values):
        acc |= (v & ((1 << w) - 1)) << (i * w)
    return acc.to_bytes((len(values) * w + 7) // 8, "little")


def delta_binary_packed(values, block: int = 128, n_mb: int = 4, count: Optional[int] = None, width: Optional[int] = None) -> bytes:
    """DELTA_BINARY_PACKED of int32 values: header, then per block the zigzag min delta, the miniblock bit widths and
    the miniblocks holding values, each whole.  `count` overrides the header's total, `width` the first bit width."""
    vals = [int(v) for v in values]
    out = _uleb(block) + _uleb(n_mb) + _uleb(len(vals) if count is None else count) + _zigzag(vals[0] if vals else 0)
    per = block // n_mb
    deltas = [vals[i] - vals[i - 1] for i in range(1, len(vals))]
    for b in range(0, len(deltas), block):
        blk = deltas[b:b + block]
        mn = min(blk)
        rel = [d - mn for d in blk]
        used = (len(rel) + per - 1) // per
        ws = [max(rel[m * per:(m + 1) * per]).bit_length() for m in range(used)] + [0] * (n_mb - used)
        if width is not None and b == 0:
            ws[0] = width
        out += _zigzag(mn) + bytes(ws)
        for m in range(used):
            mb = rel[m * per:(m + 1) * per]
            out += _pack(mb + [0] * (per - len(mb)), ws[m])
    return out


def dlba_page(values: List[bytes], lengths=None, **dbp) -> bytes:
    lens = [len(v) for v in values] if lengths is None else lengths
    return delta_binary_packed(lens, **dbp) + b"".join(values)


def dba_page(values: List[bytes], prefixes=None, suffix_lengths=None, suffix_count=None, extra: bytes = b"") -> bytes:
    pre, suf, prev = [], [], b""
    for v in values:
        k = 0
        while k < min(len(v), len(prev)) and v[k] == prev[k]:
            k += 1
        pre.append(k)
        suf.append(v[k:])
        prev = v
    pre = pre if prefixes is None else prefixes
    lens = [len(x) for x in suf] if suffix_lengths is None else suffix_lengths
    return delta_binary_packed(pre) + delta_binary_packed(lens, count=suffix_count) + b"".join(suf) + extra


def _header(ptype: int, payload_len: int, sub_fid: int, sub) -> bytes:
    return _Struct().i32(1, ptype).i32(2, payload_len).i32(3, payload_len).struct(sub_fid, sub).done()


def _data_page(enc: int, n: int, payload: bytes) -> bytes:
    return _header(PAGE_DATA, len(payload), 5, _Struct().i32(1, n).i32(2, enc).i32(3, ENC_RLE).i32(4, ENC_RLE)) + payload


def assemble(pages, dictionary: Optional[List[bytes]] = None, check: bool = True) -> bytes:
    """One row group: `s` (REQUIRED BYTE_ARRAY, UTF8) from `pages`, a list of (encoding, values, payload or None for the
    encoding's own), behind a dictionary page of `dictionary` when given; `timestamp` (REQUIRED INT64, PLAIN) 0 .. n-1.
    With `check`, pyarrow must read `s` as the pages' values."""
    out = bytearray(b"PAR1")
    n = sum(len(v) for _, v, _ in pages)
    start = len(out)
    data_off = start
    if dictionary is not None:
        d = b"".join(struct.pack("<I", len(x)) + x for x in dictionary)
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
                payload = b"".join(struct.pack("<I", len(v)) + v for v in values)
            elif enc == ENC_DLBA:
                payload = dlba_page(values)
            else:
                payload = dba_page(values)
        out += _data_page(enc, len(values), payload)
        expect += [v.decode() for v in values]
    s_size = len(out) - start
    encs = sorted({e for e, _, _ in pages} | {ENC_RLE} | ({ENC_PLAIN} if dictionary is not None else set()))
    md = (_Struct().i32(1, PT_BYTE_ARRAY).list(2, 5, [_zigzag(e) for e in encs]).list(3, 8, [_uleb(1) + b"s"]).i32(4, 0)
          .i64(5, n).i64(6, s_size).i64(7, s_size).i64(9, data_off))
    if dictionary is not None:
        md.i64(11, start)
    chunks = [_Struct().i64(2, start).struct(3, md).done()]
    t_start = len(out)
    ts = np.arange(n, dtype="<i8").tobytes()
    out += _data_page(ENC_PLAIN, n, ts)
    t_size = len(out) - t_start
    md = (_Struct().i32(1, PT_INT64).list(2, 5, [_zigzag(ENC_PLAIN), _zigzag(ENC_RLE)]).list(3, 8, [_uleb(9) + b"timestamp"])
          .i32(4, 0).i64(5, n).i64(6, t_size).i64(7, t_size).i64(9, t_start))
    chunks.append(_Struct().i64(2, t_start).struct(3, md).done())
    rgs = [_Struct().list(1, 12, chunks).i64(2, s_size + t_size).i64(3, n).done()]
    schema_els = [_Struct().binary(4, b"schema").i32(5, 2).done(),
                  _Struct().i32(1, PT_BYTE_ARRAY).i32(3, 0).binary(4, b"s").i32(6, 0).done(),
                  _Struct().i32(1, PT_INT64).i32(3, 0).binary(4, b"timestamp").done()]
    kv = [_Struct().binary(1, b"dynamic_columns").binary(2, b"").done()]
    footer = (_Struct().i32(1, 1).list(2, 12, schema_els).i64(3, n).list(4, 12, rgs).list(5, 12, kv)
              .binary(6, b"frostgpu tests (delta_strings.py)").done())
    out += footer + struct.pack("<I", len(footer)) + b"PAR1"
    buf = bytes(out)
    if check:
        t = pq.read_table(io.BytesIO(buf))
        assert t.column("s").to_pylist() == expect, "pyarrow disagrees with the pages"
        assert t.column("timestamp").to_pylist() == list(range(n))
    return buf


def mixed_values() -> List[List[bytes]]:
    """The pages of the mixed chunk: dictionary indices, DLBA, DBA, PLAIN (values in and out of the dictionary)."""
    dict_vals = [f"dict/{i:03d}".encode() for i in range(20)]
    rng = np.random.default_rng(31)
    pick = lambda pool, n: [pool[int(i)] for i in rng.integers(0, len(pool), size=n)]
    new = [f"fallback/{i:04d}/frame".encode() for i in range(300)]
    return [pick(dict_vals, 200), pick(dict_vals + new[:150], 300), sorted(pick(dict_vals + new, 500)), pick(new + dict_vals, 100)]


@functools.lru_cache(maxsize=None)
def mixed_file() -> bytes:
    """A dictionary chunk whose writer fell back part of the way through, to DLBA, DBA and PLAIN pages."""
    dict_vals = [f"dict/{i:03d}".encode() for i in range(20)]
    p = mixed_values()
    return assemble([(ENC_RLE_DICTIONARY, p[0], None), (ENC_DLBA, p[1], None), (ENC_DBA, p[2], None), (ENC_PLAIN, p[3], None)],
                    dictionary=dict_vals)


def mixed_strings() -> List[str]:
    return [v.decode() for page in mixed_values() for v in page]


def _corrupt_values():
    return [f"value/{i:03d}/{'x' * (i % 5)}".encode() for i in range(150)]


def corrupted():
    """(name, file, message) per validation rule: one DLBA or DBA page that breaks it, behind a valid PLAIN page."""
    v = _corrupt_values()
    lens = [len(x) for x in v]
    head = (ENC_PLAIN, [b"ok-1", b"ok-2"], None)
    f = lambda enc, payload: assemble([head, (enc, v, payload)], check=False)
    chain_n = 93000  # values "a", "aa", ...: one byte of suffix each, n (n + 1) / 2 bytes rebuilt
    chain = dba_prefix_only(chain_n)
    return [
        ("block_size", f(ENC_DLBA, dlba_page(v, block=64, n_mb=2)), "DELTA_LENGTH_BYTE_ARRAY lengths: DELTA_BINARY_PACKED block size is not a multiple of 128"),
        ("miniblock_size", f(ENC_DLBA, dlba_page(v, block=128, n_mb=8)), "DELTA_LENGTH_BYTE_ARRAY lengths: DELTA_BINARY_PACKED miniblock size is not a multiple of 32"),
        ("count", f(ENC_DLBA, dlba_page(v, count=len(v) + 1)), "DELTA_LENGTH_BYTE_ARRAY lengths: DELTA_BINARY_PACKED value count differs from the page's values"),
        ("bit_width", f(ENC_DLBA, dlba_page(v, width=33)), "DELTA_LENGTH_BYTE_ARRAY lengths: DELTA_BINARY_PACKED miniblock bit width > 32"),
        ("overrun", f(ENC_DLBA, delta_binary_packed(lens)[:-4]), "DELTA_LENGTH_BYTE_ARRAY lengths: DELTA_BINARY_PACKED stream overruns its page"),
        ("negative_length", f(ENC_DLBA, dlba_page(v, lengths=[-1] + lens[1:])), "DELTA_LENGTH_BYTE_ARRAY length is negative"),
        ("dlba_sum", f(ENC_DLBA, dlba_page(v) + b"!"), "DELTA_LENGTH_BYTE_ARRAY lengths do not add up to the page's value bytes"),
        ("suffix_count", f(ENC_DBA, dba_page(v, suffix_count=len(v) - 1)), "DELTA_BYTE_ARRAY suffix lengths: DELTA_BINARY_PACKED value count differs from the page's values"),
        ("negative_prefix", f(ENC_DBA, dba_page(v, prefixes=[0, -1] + [0] * (len(v) - 2))), "DELTA_BYTE_ARRAY prefix length is negative"),
        ("negative_suffix", f(ENC_DBA, dba_page(v, suffix_lengths=[-2] + [len(x) for x in v[1:]])), "DELTA_BYTE_ARRAY suffix length is negative"),
        ("first_prefix", f(ENC_DBA, dba_page(v, prefixes=[1] + [0] * (len(v) - 1))), "DELTA_BYTE_ARRAY prefix is longer than the value before it"),
        ("long_prefix", f(ENC_DBA, dba_page(v, prefixes=[0, 100] + [0] * (len(v) - 2))), "DELTA_BYTE_ARRAY prefix is longer than the value before it"),
        ("dba_sum", f(ENC_DBA, dba_page(v, extra=b"??")), "DELTA_BYTE_ARRAY suffix lengths do not add up to the page's value bytes"),
        ("rebuilt_4gib", assemble([head, (ENC_DBA, [b"a"] * chain_n, chain)], check=False), "DELTA_BYTE_ARRAY values of one chunk exceed 4 GiB"),
    ]


def dba_prefix_only(n: int) -> bytes:
    """A DBA page of n values, value i being i + 1 bytes "a": prefix i, suffix "a"."""
    return delta_binary_packed(list(range(n))) + delta_binary_packed([1] * n) + b"a" * n
