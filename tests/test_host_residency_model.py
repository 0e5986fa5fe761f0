"""The residency model (tests/residency_model.py) on the host: its reference agrees with pyarrow.compute's group-by
wherever the two semantics coincide, its fixtures hold the encodings and code widths they claim, and its sequence
generator is deterministic."""
import io

import pyarrow as pa
import pyarrow.compute as pc
import pyarrow.parquet as pq
import pytest

from frostdb_b200 import logicalplan as lp
from tests import residency_model as m


def _pyarrow_groups(parts, keys):
    """Sum / Count / Min / Max of value per key with pyarrow.compute (Sum of int64 wraps in the reference only: the
    compared parts have small values)."""
    t = pa.concat_tables([pq.read_table(io.BytesIO(m.file_of(p))).select(list(keys) + ["value"]).cast(
        pa.schema([pa.field(k, pa.string()) for k in keys] + [pa.field("value", pa.int64())])) for p in parts])
    g = t.group_by(list(keys), use_threads=False).aggregate([("value", "sum"), ("value", "count"), ("value", "min"), ("value", "max")])
    cols = [g.column(k).to_pylist() for k in keys] + [g.column(f"value_{f}").to_pylist() for f in ("sum", "count", "min", "max")]
    return {tuple(r[:len(keys)]): tuple(r[len(keys):]) for r in zip(*cols)}


@pytest.mark.parametrize("keys", [("s_dict",), ("s_plain", "s_dba"), ("s_dlba", "s_fallback")])
def test_reference_agrees_with_pyarrow_group_by(keys):
    parts = ["sorted_a", "unsorted_a", "sorted_c", "edge"]  # (no full-range values: pyarrow's sum would overflow)
    aggs = (lp.Sum(m.V), lp.Count(m.V), lp.Min(m.V), lp.Max(m.V))
    plan = m.Plan("check", "agg", keys, aggs)
    assert m.reference(plan, parts) == _pyarrow_groups(parts, keys)


def test_reference_wraps_sums_and_keeps_rows_in_order():
    plan = m.Plan("check", "agg", (), (lp.Sum(m.V), lp.Count(m.V)))
    vals = pq.read_table(io.BytesIO(m.file_of("sorted_b"))).column("value").to_pylist()
    total = sum(vals)
    assert not -(1 << 63) <= total < (1 << 63)  # the fixture's sum does leave int64
    assert m.reference(plan, ["sorted_b"]) == {(): ((total + (1 << 63)) % (1 << 64) - (1 << 63), len(vals))}
    rows = m.reference(m.Plan("rows", "rows", ("timestamp", "floatvalue", m.LABEL), (), m.V.Gt(lp.Literal(900))), ["unsorted_a", "sorted_b"])
    t = pa.concat_tables([pq.read_table(io.BytesIO(m.file_of(p))) for p in ("unsorted_a", "sorted_b")], promote_options="default")
    t = t.filter(pc.greater(t.column("value"), 900))
    exp = list(zip(t.column("timestamp").to_pylist(), t.column("floatvalue").to_pylist(), t.column(m.LABEL).to_pylist()))
    assert rows == exp and any(r[2] is None for r in rows) and any(r[2] is not None for r in rows)


@pytest.mark.parametrize("name", [s.name for s in m.SPECS])
def test_fixtures_hold_the_layouts_they_claim(name):
    buf = m.file_of(name)  # (asserts every column's encodings per row group)
    spec = m.SPEC_BY_NAME[name]
    md = pq.ParquetFile(io.BytesIO(buf)).metadata
    assert [md.row_group(g).num_rows for g in range(md.num_row_groups)] == list(spec.rgs)
    assert (m.LABEL in md.schema.names) == spec.label
    t = m.table_of(name)
    ts = t.column("timestamp").to_pylist()
    assert ts == sorted(ts)
    if spec.key == "runs":
        keys = t.column("s_dict").to_pylist()
        assert all(keys[i] == keys[i - 1] for i in range(1, len(keys)) if i % spec.run)
    f = [x for x in t.column("floatvalue").to_pylist() if x is not None]
    assert all(x * 8 == int(x * 8) for x in f) and t.column("floatvalue").null_count > 0


def test_edge_parts_hold_the_widths_and_lengths_they_claim():
    assert m.key_widths("edge", "s_plain") == [0, 1, 2, 6, 8, 8, 9, 13]
    assert m.key_widths("wide", "s_plain") == [6, 17, 12]
    assert [hi - lo for lo, hi in m.row_group_bounds("edge")] == [1, 31, 32, 33, 255, 256, 257, 4097]
    lengths = {len(v) for v in m.table_of("edge").column("s_plain").to_pylist()}
    assert set(m.LENGTHS) <= lengths
    dba = m.table_of("edge").column("s_dba").to_pylist()
    pairs = list(zip(dba, dba[1:]))
    assert any(a == b for a, b in pairs if a is not None)
    assert any(a is not None and b is not None and b.startswith(a) and a != b for a, b in pairs)
    # s_dict of the wide part: row groups whose largest first-occurrence id needs 8, 32 and 16 bits
    d = m.table_of("wide").column("s_dict").to_pylist()
    ids = {}
    for v in d:
        ids.setdefault(v, len(ids))
    top = [max(ids[v] for v in d[lo:hi]) for lo, hi in m.row_group_bounds("wide")]
    assert top[0] < 256 and top[1] >= 65536 and 256 <= top[2] < 65536


def test_sequences_are_deterministic_and_well_formed():
    a, b = m.sequence(7, 40), m.sequence(7, 40)
    assert a == b and a != m.sequence(8, 40) and len(a) == 40
    kinds = {op[0] for s in range(16) for op in m.sequence(s, 30)}
    assert kinds == {"put", "query", "decode", "drop", "corrupt", "switch"}
    for s in range(16):
        visible = []
        for op in m.sequence(s, 30):
            if op[0] == "put":
                assert op[1] not in visible and op[2] in m.HOWS
                visible.append(op[1])
            elif op[0] == "drop":
                visible.remove(op[1])
            elif op[0] == "decode":
                assert op[1] in visible and op[2] in m.table_of(op[1]).column_names


@pytest.mark.parametrize("filt", [None, m.V.Gt(lp.Literal(0)), lp.Col("s_dba").NotEq(lp.Literal(m._shared("s_dba", 500)[0]))],
                         ids=["none", "value_gt", "s_dba_ne"])
def test_distinct_reference_agrees_with_pyarrow_filter_and_unique(filt):
    parts = ["unsorted_a", "sorted_a", "edge"]
    keys = ["s_dict", "s_dlba"]
    t = pa.concat_tables([pq.read_table(io.BytesIO(m.file_of(p))).select(keys + ["value", "s_dba"]).cast(
        pa.schema([pa.field(k, pa.string()) for k in keys] + [pa.field("value", pa.int64()), pa.field("s_dba", pa.string())]))
        for p in parts])
    if filt is not None and filt.Left.Name() == "value":
        t = t.filter(pc.greater(t.column("value"), 0))
    elif filt is not None:  # (NULL != literal selects nothing)
        t = t.filter(pc.not_equal(t.column("s_dba"), filt.Right.Value))
    exp = set(zip(*[t.group_by(keys, use_threads=False).aggregate([]).column(k).to_pylist() for k in keys]))
    got = m.reference(m.Plan("d", "distinct", tuple(keys), (), filt), parts)
    assert got == exp
    if filt is not None:
        assert got < m.reference(m.Plan("d", "distinct", tuple(keys), (), None), parts)
