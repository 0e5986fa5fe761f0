"""FrostDB's dynamic-column Parquet layout, host side (test / benchmark infrastructure).

Mirrors what the reference's `dynparquet.Schema` writes (dynparquet/schema.go:508-552, 684-713,
1111-1157; samples/example.go:157-226): one flat root group, columns sorted by name, dynamic
columns flattened to `<column>.<name>` optional BYTE_ARRAY/UTF8 RLE_DICTIONARY leaves, required
INT64 PLAIN for timestamp/value, optional DOUBLE PLAIN, no compression, key-value metadata
`dynamic_columns`.  In a FrostDB process the Go side produces these bytes (table.go:1267
compactParts); here pyarrow's writer stands in for parquet-go so the files the kernels decode are
written by an independent implementation.  Nothing in here is on the GPU path.
"""
from __future__ import annotations

import dataclasses
import io
from typing import Dict, List, Optional, Sequence

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq

TYPE_STRING = "string"
TYPE_INT64 = "int64"
TYPE_DOUBLE = "double"


@dataclasses.dataclass
class ColumnDefinition:
    """schemapb.Column (name, StorageLayout{type, nullable, encoding}, dynamic)."""
    name: str
    type: str = TYPE_STRING
    nullable: bool = False
    dynamic: bool = False
    rle_dictionary: bool = False
    delta_binary_packed: bool = False  # StorageLayout_ENCODING_DELTA_BINARY_PACKED (int64 columns only)
    compression: str = "NONE"  # StorageLayout.Compression: "NONE" or "LZ4_RAW" (COMPRESSION_LZ4_RAW)


@dataclasses.dataclass
class SortingColumn:
    name: str
    descending: bool = False
    nulls_first: bool = False


@dataclasses.dataclass
class Schema:
    name: str
    columns: List[ColumnDefinition]
    sorting_columns: List[SortingColumn]

    def column(self, name: str) -> Optional[ColumnDefinition]:
        for c in self.columns:
            if c.name == name:
                return c
        return None

    def definition_for(self, concrete: str) -> ColumnDefinition:
        """Definition of a concrete column name (`labels.job` -> the dynamic `labels` column)."""
        c = self.column(concrete)
        if c is not None and not c.dynamic:
            return c
        if "." in concrete:
            base = concrete.split(".", 1)[0]
            c = self.column(base)
            if c is not None and c.dynamic:
                return c
        raise KeyError(f"column {concrete!r} is not part of schema {self.name!r}")


def SampleDefinition() -> Schema:
    """samples/example.go:157-211."""
    return Schema(
        name="test",
        columns=[
            ColumnDefinition("example_type", TYPE_STRING, rle_dictionary=True),
            ColumnDefinition("labels", TYPE_STRING, nullable=True, dynamic=True, rle_dictionary=True),
            ColumnDefinition("stacktrace", TYPE_STRING, rle_dictionary=True),
            ColumnDefinition("timestamp", TYPE_INT64),
            ColumnDefinition("value", TYPE_INT64),
        ],
        sorting_columns=[
            SortingColumn("example_type"),
            SortingColumn("labels", nulls_first=True),
            SortingColumn("timestamp"),
            SortingColumn("stacktrace", nulls_first=True),
        ],
    )


def BytesDefinition() -> Schema:
    """The logictest "bytes" schema (logictest/logic_test.go:110-142): dynamic labels, timestamp, and a non-dynamic
    string column `value`.  Upstream stores `timestamp` as UINT64 and `value` as DELTA_LENGTH_BYTE_ARRAY + LZ4_RAW;
    this mirror writes int64 and RLE_DICTIONARY (the engine takes neither compressed pages nor non-dictionary strings
    in Parquet parts) — the logical column types, which is what the queries see, are the same."""
    return Schema(
        name="test",
        columns=[
            ColumnDefinition("labels", TYPE_STRING, nullable=True, dynamic=True, rle_dictionary=True),
            ColumnDefinition("timestamp", TYPE_INT64),
            ColumnDefinition("value", TYPE_STRING, rle_dictionary=True),
        ],
        sorting_columns=[
            SortingColumn("labels", nulls_first=True),
            SortingColumn("timestamp"),
            SortingColumn("value"),
        ],
    )


def SampleDefinitionWithFloat() -> Schema:
    """samples/example.go:215-226."""
    s = SampleDefinition()
    s.columns.append(ColumnDefinition("floatvalue", TYPE_DOUBLE, nullable=True))
    return s


_CODECS = {"NONE": "NONE", "LZ4_RAW": "LZ4"}


def _arrow_column(defn: ColumnDefinition, values, n_rows: int) -> pa.Array:
    if isinstance(values, (pa.Array, pa.ChunkedArray)):
        return values
    if defn.type == TYPE_STRING:
        if isinstance(values, tuple):  # (indices int32 with -1 = NULL, dictionary list[str])
            idx, dictionary = values
            idx = np.asarray(idx, dtype=np.int32)
            mask = idx < 0
            ind = pa.array(np.where(mask, 0, idx), type=pa.int32(), mask=mask if mask.any() else None)
            return pa.DictionaryArray.from_arrays(ind, pa.array(dictionary, type=pa.string()))
        arr = pa.array(list(values), type=pa.string())
        return arr.dictionary_encode() if defn.rle_dictionary else arr
    if defn.type == TYPE_INT64:
        if isinstance(values, np.ndarray):
            return pa.array(values.astype(np.int64, copy=False))
        return pa.array(list(values), type=pa.int64())
    if defn.type == TYPE_DOUBLE:
        if isinstance(values, np.ndarray):
            return pa.array(values.astype(np.float64, copy=False))
        return pa.array(list(values), type=pa.float64())
    raise ValueError(defn.type)


def sort_permutation(schema: Schema, columns: Dict[str, object], n_rows: int) -> np.ndarray:
    """Row order compaction would produce: schema sorting columns, dynamic columns expanded in
    name order, NULLs first where the schema says so (dynparquet/schema.go ParquetSortingColumns)."""
    keys = []  # least significant last for np.lexsort -> build most significant first, reverse later
    for sc in schema.sorting_columns:
        defn = schema.column(sc.name)
        names = sorted(n for n in columns if n.startswith(sc.name + ".")) if defn is not None and defn.dynamic else (
            [sc.name] if sc.name in columns else [])
        for n in names:
            v = columns[n]
            if isinstance(v, tuple):
                idx, dictionary = v
                order = np.argsort(np.argsort(np.asarray(dictionary, dtype=object)))
                rank = np.where(np.asarray(idx) < 0, -1, order[np.maximum(np.asarray(idx), 0)])
                if not sc.nulls_first:
                    rank = np.where(rank < 0, len(dictionary), rank)
                keys.append(-rank if sc.descending else rank)
            elif isinstance(v, np.ndarray) and v.dtype.kind in "if":
                keys.append(-v if sc.descending else v)
            else:
                lst = list(v)
                uniq = sorted({x for x in lst if x is not None})
                pos = {x: i for i, x in enumerate(uniq)}
                null_rank = -1 if sc.nulls_first else len(uniq)
                rank = np.array([null_rank if x is None else pos[x] for x in lst], dtype=np.int64)
                keys.append(-rank if sc.descending else rank)
    if not keys:
        return np.arange(n_rows)
    return np.lexsort(tuple(reversed(keys)))


def write_part(schema: Schema, columns: Dict[str, object], *, sort: bool = True,
               row_group_size: Optional[int] = None, data_page_size: Optional[int] = None,
               data_page_version: str = "2.0", dictionary_pagesize_limit: Optional[int] = None,
               write_statistics: bool = True) -> bytes:
    """Serialises one part.  `columns` maps concrete column names (`labels.job`, `timestamp`, ...)
    to values: list (None = NULL), numpy array, or (indices, dictionary) for dictionary strings."""
    names = sorted(columns)  # the reference sorts columns by name (dynparquet/schema.go newSchema)
    if not names:
        raise ValueError("no columns")
    n_rows = None
    for n in names:
        v = columns[n]
        ln = len(v[0]) if isinstance(v, tuple) else len(v)
        if n_rows is None:
            n_rows = ln
        elif ln != n_rows:
            raise ValueError(f"column {n} has {ln} rows, expected {n_rows}")
    perm = sort_permutation(schema, columns, n_rows) if sort and n_rows > 1 else None
    fields, arrays, dict_cols, plain_cols, codecs = [], [], [], {}, {}
    dyn: Dict[str, List[str]] = {}
    for n in names:
        defn = schema.definition_for(n)
        v = columns[n]
        if perm is not None:
            if isinstance(v, tuple):
                v = (np.asarray(v[0])[perm], v[1])
            elif isinstance(v, np.ndarray):
                v = v[perm]
            else:
                lst = list(v)
                v = [lst[i] for i in perm]
        arr = _arrow_column(defn, v, n_rows)
        nullable = defn.nullable
        if not nullable and arr.null_count:
            raise ValueError(f"column {n} is not nullable but has NULLs")
        if defn.delta_binary_packed and defn.type != TYPE_INT64:
            raise ValueError(f"column {n}: DELTA_BINARY_PACKED needs an int64 column, not {defn.type}")
        if defn.type == TYPE_STRING and defn.rle_dictionary:
            dict_cols.append(n)
        else:
            plain_cols[n] = "DELTA_BINARY_PACKED" if defn.delta_binary_packed else "PLAIN"
        if defn.compression not in _CODECS:
            raise ValueError(f"column {n}: compression {defn.compression!r} is not one of {sorted(_CODECS)}")
        codecs[n] = _CODECS[defn.compression]
        if defn.dynamic:
            dyn.setdefault(defn.name, []).append(n.split(".", 1)[1])
        fields.append(pa.field(n, arr.type, nullable=nullable))
        arrays.append(arr)
    table = pa.Table.from_arrays(arrays, schema=pa.schema(fields))
    # dynparquet/dynamiccolumns.go:11-39: "labels:a,b;other:c"
    kv = ";".join(f"{k}:{','.join(sorted(v))}" for k, v in sorted(dyn.items()))
    table = table.replace_schema_metadata({"dynamic_columns": kv})
    sink = io.BytesIO()
    kwargs = {}
    if data_page_size is not None:
        kwargs["data_page_size"] = data_page_size
    if dictionary_pagesize_limit is not None:
        kwargs["dictionary_pagesize_limit"] = dictionary_pagesize_limit
    # (pyarrow's "lz4" is Parquet's LZ4_RAW, codec 7; every column uncompressed keeps the one-codec call)
    compression = codecs if any(c != "NONE" for c in codecs.values()) else "NONE"
    pq.write_table(table, sink, compression=compression, use_dictionary=dict_cols,
                   column_encoding=plain_cols or None, data_page_version=data_page_version,
                   row_group_size=row_group_size or max(n_rows, 1), write_statistics=write_statistics,
                   store_schema=False, **kwargs)
    return sink.getvalue()


def read_part(buf: bytes) -> pa.Table:
    """Independent decode (pyarrow) of a part, for cross-checks."""
    return pq.read_table(io.BytesIO(buf))
