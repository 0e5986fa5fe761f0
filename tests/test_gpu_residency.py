"""Making columns resident (upload_columns in residency.cpp) on borrowed parts, where nothing goes to the device until a
query needs it:
- one Execute over a table of several parts, each mixing PLAIN, DELTA_LENGTH_BYTE_ARRAY, DELTA_BYTE_ARRAY and
  dictionary string columns with a DELTA_BINARY_PACKED int64 column, interns the parts' strings together and gives
  what the same parts put eagerly give, and pyarrow's answer;
- a plan refused on an unreadable column uploads nothing behind it: the next plan that reads those columns copies
  their bytes;
- a column decode_column made resident is not copied again by an Execute: that Execute copies what it copies on
  the same part put eagerly."""
import io
import re

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

from frostdb_b200 import _lib
from frostdb_b200 import dynparquet as dp
from frostdb_b200 import logicalplan as lp
from frostdb_b200 import query
from tests import delta_int64 as di
from tests import numeric_edges as ne
from tests.test_gpu_delta_int64 import two_columns
from tests.test_gpu_plain_strings import as_strings, stats_of

pytestmark = pytest.mark.gpu

STRINGS = ["a_dict", "b_plain", "c_dlba", "d_dba"]
ENCODING = {"b_plain": "PLAIN", "c_dlba": "DELTA_LENGTH_BYTE_ARRAY", "d_dba": "DELTA_BYTE_ARRAY", "value": "DELTA_BINARY_PACKED"}
V, T = lp.Col("value"), lp.Col("timestamp")
AGGS = [lp.Sum(V), lp.Count(V), lp.Min(T)]
SCHEMA = dp.Schema(name="residency",
                   columns=[dp.ColumnDefinition(s, dp.TYPE_STRING, nullable=True) for s in STRINGS]
                   + [dp.ColumnDefinition("timestamp", dp.TYPE_INT64), dp.ColumnDefinition("value", dp.TYPE_INT64, delta_binary_packed=True)],
                   sorting_columns=[dp.SortingColumn("timestamp")])


def mixed_part(seed: int, n: int = 6000) -> pa.Table:
    """Values from pools whose entries share long prefixes (front coding), each part drawing on its own pool too, so
    that the parts add new strings to each other's columns."""
    rng = np.random.default_rng(seed)
    def strings(k, hi, p_null):
        pool = [f"/srv/app/{k}/module_{i % 50:04d}/frame_{i}" for i in range(hi)] + [f"part{seed}/{k}/{i}" for i in range(20)]
        idx = rng.integers(0, len(pool), n)
        return pa.array([None if x else pool[i] for i, x in zip(idx, rng.random(n) < p_null)], type=pa.string())
    cols = {k: strings(k, hi, p) for k, hi, p in (("a_dict", 30, 0.0), ("b_plain", 200, 0.05), ("c_dlba", 500, 0.0), ("d_dba", 90, 0.1))}
    cols["timestamp"] = pa.array(np.arange(seed * n, (seed + 1) * n, dtype=np.int64))
    cols["value"] = pa.array(rng.integers(-1000, 1000, n))
    return pa.table(cols).replace_schema_metadata({"dynamic_columns": ""})


def file_of(t: pa.Table) -> bytes:
    sink = io.BytesIO()
    pq.write_table(t, sink, compression="NONE", row_group_size=2000, data_page_size=1024, use_dictionary=["a_dict"],
                   column_encoding=ENCODING, store_schema=False)
    buf = sink.getvalue()
    md = pq.ParquetFile(io.BytesIO(buf)).metadata
    for c, enc in ENCODING.items():  # the file holds the layouts it is meant to test
        i = md.schema.names.index(c)
        assert all(enc in md.row_group(g).column(i).encodings for g in range(md.num_row_groups)), (c, enc)
    return buf


def put(store, db, table, bufs, borrow, keep):
    if table in db.tables:
        store.engine.drop_table(table)
    db.Table(table, SCHEMA)
    for buf in bufs:
        arr = np.frombuffer(buf, dtype=np.uint8)
        if borrow:
            keep.append(arr)
        store.engine.put_parquet(table, arr, borrow=borrow)


def drop(store, db, *tables):
    for t in tables:
        store.engine.drop_table(t)
        db.tables.pop(t, None)


def agg(db, table, keys, aggs):
    out = []
    query.NewEngine(None, db.TableProvider()).ScanTable(table).Aggregate(aggs, [lp.Col(k) for k in keys]).Execute(None, lambda c, r: out.append(r))
    return ne.result_map(out, keys, aggs)


def test_one_execute_interns_every_part_of_a_borrowed_table(store):
    db = store.DB(None, "residency")
    parts = [mixed_part(s) for s in (1, 2, 3)]
    bufs = [file_of(t) for t in parts]
    exp = {}
    for t in parts:
        for r in t.to_pylist():
            k = tuple(r[c] for c in STRINGS)
            s, n, m = exp.get(k, (0, 0, r["timestamp"]))
            exp[k] = (s + r["value"], n + 1, min(m, r["timestamp"]))
    keep = []
    try:
        put(store, db, "res_borrow", bufs, True, keep)
        put(store, db, "res_eager", bufs, False, keep)
        assert stats_of(store, "res_borrow", None, STRINGS, AGGS)["h2d_bytes"] > 0
        got = agg(db, "res_borrow", STRINGS, AGGS)
        assert got == agg(db, "res_eager", STRINGS, AGGS)
        assert got == exp
        for k in STRINGS:
            assert store.engine.dict_export("res_borrow", k) == store.engine.dict_export("res_eager", k), k
    finally:
        drop(store, db, "res_borrow", "res_eager")


def test_a_refused_plan_leaves_the_columns_behind_its_refusal_on_the_host(store):
    """Part 0's `value` is unreadable and comes first in residency order: part 1's `value` stays on the host until a
    plan reads it with part 0 gone, and that plan copies what it copies on a table of part 1 alone."""
    _, bad, message = next(c for c in di.corrupted() if c[0] == "bit_width")
    _, good, exp = di.hand_layouts()[0]
    db = store.DB(None, "residency")
    keep = []
    try:
        for t in ("res_refused", "res_alone"):
            if t in db.tables:
                store.engine.drop_table(t)
            db.Table(t, two_columns())
        for table, bufs in (("res_refused", [bad, good]), ("res_alone", [good])):
            for buf in bufs:
                arr = np.frombuffer(buf, dtype=np.uint8)
                keep.append(arr)
                store.engine.put_parquet(table, arr, borrow=True)
        with pytest.raises(_lib.FrostGPUError, match=re.escape("column value: " + message)) as e:
            agg(db, "res_refused", [], [lp.Sum(V)])
        assert e.value.code == _lib.FGPU_ERR_UNSUPPORTED
        store.engine.drop_part("res_refused", 0)
        alone = stats_of(store, "res_alone", None, [], [lp.Sum(V)])["h2d_bytes"]
        assert alone > 0
        assert stats_of(store, "res_refused", None, [], [lp.Sum(V)])["h2d_bytes"] == alone
        s = (sum(exp) + (1 << 63)) % (1 << 64) - (1 << 63)
        assert agg(db, "res_refused", [], [lp.Sum(V)]) == {(): (s,)}
    finally:
        drop(store, db, "res_refused", "res_alone")


def test_decode_column_leaves_the_column_resident(store):
    t = mixed_part(4)
    buf = file_of(t)
    db = store.DB(None, "residency")
    keep = []
    filt = lp.And(lp.Col("d_dba").NotEq(lp.Literal("absent")), V.Gt(lp.Literal(-5000)))
    h2d = {}
    try:
        for table, borrow in (("res_fresh", True), ("res_decoded", True), ("res_eager", False)):
            put(store, db, table, [buf], borrow, keep)
        assert as_strings(store.engine.decode_column("res_decoded", 0, "d_dba")) == t.column("d_dba").to_pylist()
        assert store.engine.decode_column("res_decoded", 0, "value").to_pylist() == t.column("value").to_pylist()
        for table in ("res_fresh", "res_decoded", "res_eager"):  # (every Execute also uploads its plan's descriptors)
            h2d[table] = stats_of(store, table, filt, ["d_dba", "value"], [], kind=_lib.PLAN_FILTER)["h2d_bytes"]
    finally:
        drop(store, db, "res_fresh", "res_decoded", "res_eager")
    assert h2d["res_decoded"] == h2d["res_eager"] < h2d["res_fresh"], h2d
