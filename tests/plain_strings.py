"""Parquet parts whose string column `s` is written without a dictionary (PLAIN BYTE_ARRAY pages), or with a dictionary
whose writer falls back to PLAIN part of the way through, each with an RLE_DICTIONARY twin holding the same rows.

Every layout has the columns `s` (string, the column under test), `timestamp` (int64, unique), `value` (int64) and
`fvalue` (double, nullable).  The values are ASCII, so the host description (which escapes bytes >= 0x7f) prints them
as pyarrow reads them."""
import dataclasses
import functools
import io
from typing import List, Optional

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq

from frostdb_b200 import dynparquet as dp

CK_DICT_STR = 2


@dataclasses.dataclass(frozen=True)
class Layout:
    name: str
    n_rows: int
    seed: int
    version: str = "2.0"        # data page version
    nullable: bool = False
    null_p: float = 0.0         # NULL rate of `s`
    n_distinct: int = 50
    min_len: int = 1
    max_len: int = 24
    empty_p: float = 0.0        # rate of empty strings
    null_head: int = 0          # the first rows of `s` are NULL (with row_group_size == null_head: an all-NULL chunk)
    row_group_size: Optional[int] = None
    data_page_size: Optional[int] = None
    write_batch_size: Optional[int] = None
    fallback: bool = False      # dictionary chunk with a small dictionary page limit: the writer falls back to PLAIN
    collisions: bool = False    # values sharing their first bytes, differing in length


LAYOUTS = [
    Layout("v1_required", 6000, 1, version="1.0", row_group_size=4000, data_page_size=2048),
    Layout("v2_required", 6000, 2, row_group_size=4000, data_page_size=2048),
    Layout("v1_optional", 6000, 3, version="1.0", nullable=True, null_p=0.2, data_page_size=4096),
    Layout("v2_optional", 6000, 4, nullable=True, null_p=0.3, row_group_size=2500, data_page_size=4096),
    Layout("all_null_chunk", 3000, 5, nullable=True, null_p=0.1, null_head=1000, row_group_size=1000),
    Layout("empty_and_long", 3000, 6, nullable=True, null_p=0.1, n_distinct=400, min_len=1, max_len=5000, empty_p=0.2),
    Layout("many_small_pages", 5000, 7, nullable=True, null_p=0.05, data_page_size=64, write_batch_size=16),
    Layout("one_row", 1, 8),
    Layout("fallback_v1", 20000, 9, version="1.0", n_distinct=6000, fallback=True, row_group_size=12000),
    Layout("fallback_v2", 20000, 10, nullable=True, null_p=0.1, n_distinct=6000, fallback=True),
    Layout("collisions", 30000, 11, n_distinct=20000, collisions=True),
]
LAYOUT_BY_NAME = {l.name: l for l in LAYOUTS}
NAMES = [l.name for l in LAYOUTS]


def schema() -> dp.Schema:
    return dp.Schema(
        name="plain_strings",
        columns=[
            dp.ColumnDefinition("s", dp.TYPE_STRING, nullable=True),
            dp.ColumnDefinition("timestamp", dp.TYPE_INT64),
            dp.ColumnDefinition("value", dp.TYPE_INT64),
            dp.ColumnDefinition("fvalue", dp.TYPE_DOUBLE, nullable=True),
        ],
        sorting_columns=[dp.SortingColumn("timestamp")],
    )


def _pool(l: Layout, rng) -> List[str]:
    if l.collisions:  # one prefix at every length, then many distinct values of varying length
        head = ["x" * k for k in range(0, 300)] + ["xy" * k for k in range(1, 100)]
        rest = [f"x{i:07d}" + "z" * (i % 13) for i in range(l.n_distinct - len(head))]
        return head + rest
    out, seen = [], set()
    while len(out) < l.n_distinct:
        n = int(rng.integers(l.min_len, l.max_len + 1))
        v = "".join(chr(c) for c in rng.integers(0x21, 0x7f, size=n))
        if v not in seen:
            seen.add(v)
            out.append(v)
    return out


@functools.lru_cache(maxsize=None)
def table(name: str) -> pa.Table:
    l = LAYOUT_BY_NAME[name]
    rng = np.random.default_rng(l.seed)
    pool = _pool(l, rng)
    if l.collisions:  # every value at least once, in a shuffled order
        idx = np.concatenate([rng.permutation(len(pool)), rng.integers(0, len(pool), size=max(0, l.n_rows - len(pool)))])[: l.n_rows]
    else:  # skewed, so that first occurrences spread over the chunk
        idx = np.minimum((rng.pareto(1.2, size=l.n_rows) * 3).astype(np.int64), len(pool) - 1)
    s = [pool[i] for i in idx]
    if l.empty_p:
        s = [("" if e else v) for v, e in zip(s, rng.random(l.n_rows) < l.empty_p)]
    nulls = rng.random(l.n_rows) < l.null_p
    nulls[: l.null_head] = True
    s = [None if n else v for v, n in zip(s, nulls)]
    ts = np.arange(l.n_rows, dtype=np.int64)
    value = rng.integers(-1000, 1000, size=l.n_rows)
    fv = rng.normal(size=l.n_rows) * 100.0
    fmask = rng.random(l.n_rows) < 0.1
    fields = [pa.field("fvalue", pa.float64(), nullable=True), pa.field("s", pa.string(), nullable=l.nullable),
              pa.field("timestamp", pa.int64(), nullable=False), pa.field("value", pa.int64(), nullable=False)]
    arrays = [pa.array(fv, mask=fmask), pa.array(s, type=pa.string()), pa.array(ts), pa.array(value)]
    t = pa.Table.from_arrays(arrays, schema=pa.schema(fields))
    return t.replace_schema_metadata({"dynamic_columns": ""})


def _write(name: str, dictionary: bool) -> bytes:
    l = LAYOUT_BY_NAME[name]
    kwargs = {}
    if l.data_page_size is not None:
        kwargs["data_page_size"] = l.data_page_size
    if l.write_batch_size is not None:
        kwargs["write_batch_size"] = l.write_batch_size
    if dictionary:
        kwargs["dictionary_pagesize_limit"] = 1 << 28
    elif l.fallback:
        kwargs["dictionary_pagesize_limit"] = 4096
    sink = io.BytesIO()
    pq.write_table(table(name), sink, compression="NONE", use_dictionary=["s"] if (dictionary or l.fallback) else False,
                   data_page_version=l.version, row_group_size=l.row_group_size or max(l.n_rows, 1), store_schema=False, **kwargs)
    return sink.getvalue()


@functools.lru_cache(maxsize=None)
def file_of(name: str) -> bytes:
    """The layout itself: `s` PLAIN, or dictionary with PLAIN fallback."""
    return _write(name, dictionary=False)


@functools.lru_cache(maxsize=None)
def twin_of(name: str) -> bytes:
    """The same rows with `s` RLE_DICTIONARY throughout."""
    return _write(name, dictionary=True)


def record_of(name: str) -> pa.RecordBatch:
    """The same rows as one Arrow record with `s` a plain (non-dictionary) binary array."""
    t = table(name).combine_chunks()
    cols = [t.column(n).chunk(0) if t.num_rows else pa.array([], t.schema.field(n).type) for n in t.schema.names]
    cols = [c.cast(pa.binary()) if n == "s" else c for n, c in zip(t.schema.names, cols)]
    return pa.RecordBatch.from_arrays(cols, names=t.schema.names)


def s_encodings(buf: bytes) -> List[set]:
    """The encodings the footer lists for `s`, per row group."""
    md = pq.ParquetFile(io.BytesIO(buf)).metadata
    col = md.schema.names.index("s")
    return [set(md.row_group(g).column(col).encodings) for g in range(md.num_row_groups)]


def row_group_slices(buf: bytes):
    md = pq.ParquetFile(io.BytesIO(buf)).metadata
    out, s = [], 0
    for g in range(md.num_row_groups):
        n = md.row_group(g).num_rows
        out.append((s, s + n))
        s += n
    return out


def first_occurrence(values) -> List[str]:
    seen, out = set(), []
    for v in values:
        if v is not None and v not in seen:
            seen.add(v)
            out.append(v)
    return out
