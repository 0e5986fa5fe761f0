"""DELTA_BINARY_PACKED int64 column chunks on the device (k_dbp_local, k_dbp_carry, k_dbp_add in delta_int64.cu): every
layout of tests/delta_int64.py is put eagerly and borrowed, next to its PLAIN twin and the same rows as an Arrow part,
and then
- decode_column equals pyarrow's read, for the hand-assembled layouts too;
- Sum / Count / Min / Max of `value` by labels.a, labels.b under timestamp ranges, the numeric-edge literals on `value`
  and an OR filter equal the twin's and numeric_edges' reference, and the steady Execute takes the twin's kernels
  (fgpu_stats) on the sorted-run, prefix, tile and general scan paths, in hash mode and in filter-only plans;
- `value` as a group key, and a table of a DELTA_BINARY_PACKED, a PLAIN and an Arrow part;
- the first Execute over a borrowed sorted part that reads `timestamp` only copies under a quarter of the twin's bytes;
- a corrupted chunk fails only the queries that touch its column."""
import os
import re

import numpy as np
import pytest

from frostdb_b200 import _lib
from frostdb_b200 import dynparquet as dp
from frostdb_b200 import logicalplan as lp
from frostdb_b200 import query
from tests import delta_int64 as di
from tests import numeric_edges as ne
from tests.test_gpu_plain_strings import SWITCHES, stats_of

pytestmark = pytest.mark.gpu

KINDS = ["eager", "borrow", "twin", "arrow"]
V, T = lp.Col("value"), lp.Col("timestamp")
AGGS = ne.AGG_INT
PATHS = [{}, {"FROSTGPU_NO_RUNS": "1"}, {"FROSTGPU_NO_RUNS": "1", "FROSTGPU_NO_TILE": "1"},
         {"FROSTGPU_NO_RUNS": "1", "FROSTGPU_NO_TILE": "1", "FROSTGPU_NO_FAST": "1"}]
ROUTE = ("row_groups", "row_groups_pruned", "row_groups_runs", "row_groups_tiles", "row_groups_prefix", "kernel_launches")


@pytest.fixture(autouse=True)
def clean_switches():
    yield
    for k in SWITCHES:
        os.environ.pop(k, None)


def _fresh(store, db, table, schema):
    if table in db.tables:
        store.engine.drop_table(table)
    db.Table(table, schema)


def _put(store, table, buf, borrow, keep):
    arr = np.frombuffer(buf, dtype=np.uint8)
    if borrow:
        keep.append(arr)
    store.engine.put_parquet(table, arr, borrow=borrow)


@pytest.fixture(scope="module")
def parts(store):
    """Every layout as four tables of one part each: the delta file put eagerly and borrowed, the PLAIN twin, the Arrow
    record."""
    db = store.DB(None, "delta_int64")
    keep, made = [], {}
    for name in di.NAMES:
        l = di.LAYOUT_BY_NAME[name]
        for kind in KINDS:
            table = f"dbp_{name}_{kind}"
            _fresh(store, db, table, di.schema(di.columns(name), delta=kind != "twin", nullable_value=l.nullable))
            if kind == "arrow":
                store.engine.put_arrow(table, di.record_of(name))
            else:
                _put(store, table, di.twin_of(name) if kind == "twin" else di.file_of(name), kind == "borrow", keep)
            made[(name, kind)] = table
    yield db, made
    for table in made.values():
        store.engine.drop_table(table)
        db.tables.pop(table, None)


def agg(db, table, filt, keys, aggs, switches=None):
    os.environ.update(switches or {})
    try:
        out = []
        q = query.NewEngine(None, db.TableProvider()).ScanTable(table)
        (q.Filter(filt) if filt is not None else q).Aggregate(aggs, [lp.Col(k) for k in keys]).Execute(None, lambda c, r: out.append(r))
        return ne.result_map(out, keys, aggs)
    finally:
        for k in switches or {}:
            os.environ.pop(k)


def route(store, table, filt, keys, aggs, switches=None, kind=_lib.PLAN_AGGREGATE):
    """fgpu_stats of a steady Execute (the columns resident): which kernels took the row groups."""
    os.environ.update(switches or {})
    try:
        stats_of(store, table, filt, keys, aggs, kind=kind)
        st = stats_of(store, table, filt, keys, aggs, kind=kind)
        return {k: st[k] for k in ROUTE}
    finally:
        for k in switches or {}:
            os.environ.pop(k)


def ts_filters(name):
    """timestamp ranges: halves of two row groups, every row, no row."""
    rg, n = di.LAYOUT_BY_NAME[name].rg, len(di.columns(name)["timestamp"])
    return [lp.And(T.GtEq(lp.Literal(rg // 2)), T.Lt(lp.Literal(rg + rg // 2))),
            lp.And(T.GtEq(lp.Literal(0)), T.Lt(lp.Literal(n))),
            T.GtEq(lp.Literal(n + 10))]


def or_filter():
    return lp.Or(V.Lt(lp.Literal(-1)), T.Lt(lp.Literal(100)))


def edge_filters():
    return [ne.leaf(ne.V, op, x) for op in ne.OPS for x in ne.EDGE_LITERALS]


@pytest.mark.parametrize("kind", ["eager", "borrow"])
@pytest.mark.parametrize("name", di.NAMES)
def test_decode_column_matches_pyarrow(store, parts, name, kind):
    _, made = parts
    t = dp.read_part(di.twin_of(name))
    for col in ("timestamp", "value"):
        got = store.engine.decode_column(made[(name, kind)], 0, col)
        assert got.to_pylist() == t.column(col).to_pylist(), (name, kind, col)


def two_columns() -> dp.Schema:
    """The schema of the hand-assembled files: `timestamp` and `value`."""
    return dp.Schema(name="assembled", columns=[dp.ColumnDefinition("timestamp", dp.TYPE_INT64),
                                                dp.ColumnDefinition("value", dp.TYPE_INT64, delta_binary_packed=True)],
                     sorting_columns=[dp.SortingColumn("timestamp")])


@pytest.mark.parametrize("borrow", [False, True])
def test_hand_assembled_pages(store, borrow):
    """PLAIN and delta pages in one chunk, pages of 0 and 1 values, other block sizes, unused miniblocks wider than 64
    bits, bytes behind a stream: decode_column, and Sum / Count / Min / Max on the general scan kernel."""
    db = store.DB(None, "delta_int64")
    keep = []
    for name, buf, exp in di.hand_layouts():
        table = f"dbp_hand_{name}_{int(borrow)}"
        _fresh(store, db, table, two_columns())
        try:
            _put(store, table, buf, borrow, keep)
            assert store.engine.decode_column(table, 0, "value").to_pylist() == exp, name
            aggs = [lp.Sum(V), lp.Count(V), lp.Min(V), lp.Max(V)]
            s = (sum(exp) + (1 << 63)) % (1 << 64) - (1 << 63)
            assert agg(db, table, None, [], aggs) == {(): (s, len(exp), min(exp), max(exp))}, name
        finally:
            store.engine.drop_table(table)
            db.tables.pop(table, None)


@pytest.mark.parametrize("name", di.NAMES)
def test_aggregates_equal_the_twin_and_the_reference(store, parts, name):
    db, made = parts
    phys = [ne.physical(di.columns(name))]
    keys = ["value"] if name.startswith("int_key") else ne.KEYS
    for filt in [None] + ts_filters(name) + [or_filter()]:
        exp = ne.reference(phys, filt, keys, AGGS)
        what = f"{name} {filt.Name() if filt is not None else None}"
        for sw in PATHS:
            for kind in KINDS:
                ne.assert_same_result(agg(db, made[(name, kind)], filt, keys, AGGS, sw), exp, AGGS, f"{what} {kind} {sw}")
            for kind in ("eager", "borrow"):
                assert route(store, made[(name, kind)], filt, keys, AGGS, sw) == route(store, made[(name, "twin")], filt, keys, AGGS, sw), \
                    f"{what} {kind} {sw}"
    for filt in edge_filters():
        exp = ne.reference(phys, filt, keys, AGGS)
        for kind in KINDS:
            ne.assert_same_result(agg(db, made[(name, kind)], filt, keys, AGGS), exp, AGGS, f"{name} {filt.Name()} {kind}")
        assert route(store, made[(name, "eager")], filt, keys, AGGS) == route(store, made[(name, "twin")], filt, keys, AGGS), filt.Name()


@pytest.mark.parametrize("name", ["sorted", "sorted_v1", "page_edges"])
def test_sorted_parts_take_the_twins_run_and_prefix_paths(store, parts, name):
    """All-pass row groups with Sum and Count (k_runs_prefix) and filtered sorted row groups (k_runs_tma)."""
    db, made = parts
    aggs = [lp.Sum(V), lp.Count(V)]
    phys = [ne.physical(di.columns(name))]
    for filt in [None] + ts_filters(name):
        r = route(store, made[(name, "eager")], filt, ne.KEYS, aggs)
        assert r == route(store, made[(name, "twin")], filt, ne.KEYS, aggs), (name, filt)
        assert r == route(store, made[(name, "borrow")], filt, ne.KEYS, aggs), (name, filt)
        ne.assert_same_result(agg(db, made[(name, "eager")], filt, ne.KEYS, aggs), ne.reference(phys, filt, ne.KEYS, aggs), aggs, name)


@pytest.mark.parametrize("name", di.NAMES)
def test_filter_only_plans(store, parts, name):
    """Filter-only plans projecting `timestamp` and `value` (the ordered take kernels, and k_rows without them)."""
    db, made = parts
    phys = ne.physical(di.columns(name))
    valid = phys.get("value#valid")
    names = ["timestamp", "value"]
    for filt in ts_filters(name)[:1] + [or_filter(), ne.leaf(ne.V, lp.OpGt, 0)]:
        sel = np.flatnonzero(ne.selection(phys, filt))  # (a NULL `value` is projected as NULL)
        exp = [(int(phys["timestamp"][i]), int(phys["value"][i]) if valid is None or valid[i] else None) for i in sel]
        for sw in ({}, {"FROSTGPU_NO_TAKE": "1"}):
            for kind in ("eager", "borrow", "twin"):
                os.environ.update(sw)
                try:
                    out = []
                    query.NewEngine(None, db.TableProvider()).ScanTable(made[(name, kind)]).Filter(filt) \
                        .Project(*[lp.Col(n) for n in names]).Execute(None, lambda c, r: out.append(r))
                finally:
                    for k in sw:
                        os.environ.pop(k)
                ne.assert_same_rows(ne.record_rows(out, names), exp, f"{name} {kind} {filt.Name()} {sw}")
            assert route(store, made[(name, "eager")], filt, names, [], sw, kind=_lib.PLAN_FILTER) == \
                route(store, made[(name, "twin")], filt, names, [], sw, kind=_lib.PLAN_FILTER), (name, filt.Name(), sw)


def test_delta_plain_and_arrow_parts_in_one_table(store):
    """A DELTA_BINARY_PACKED, a PLAIN and an Arrow part give what three PLAIN parts give."""
    db = store.DB(None, "delta_int64")
    names = ["sorted", "unsorted", "wrap"]
    sch = di.schema(di.columns("sorted"), delta=True)
    mixed, plain, keep = "dbp_table_mixed", "dbp_table_plain", []
    try:
        _fresh(store, db, mixed, sch)
        _put(store, mixed, di.file_of(names[0]), False, keep)
        _put(store, mixed, di.twin_of(names[1]), False, keep)
        store.engine.put_arrow(mixed, di.record_of(names[2]))
        _fresh(store, db, plain, sch)
        for n in names:
            _put(store, plain, di.twin_of(n), False, keep)
        phys = [ne.physical(di.columns(n)) for n in names]
        for filt in [None, or_filter()] + ts_filters("sorted")[:1]:
            exp = ne.reference(phys, filt, ne.KEYS, AGGS)
            ne.assert_same_result(agg(db, mixed, filt, ne.KEYS, AGGS), exp, AGGS, "mixed")
            ne.assert_same_result(agg(db, plain, filt, ne.KEYS, AGGS), exp, AGGS, "plain")
    finally:
        for t in (mixed, plain):
            store.engine.drop_table(t)
            db.tables.pop(t, None)


def test_first_execute_of_a_borrowed_sorted_part_copies_a_fraction_of_the_twins_bytes(store):
    db = store.DB(None, "delta_int64")
    keep, h2d = [], {}
    n = len(di.columns("sorted")["timestamp"])
    filt = lp.And(T.GtEq(lp.Literal(100)), T.Lt(lp.Literal(n - 100)))
    for kind, buf in (("delta", di.file_of("sorted")), ("twin", di.twin_of("sorted"))):
        table = f"dbp_h2d_{kind}"
        _fresh(store, db, table, di.schema(di.columns("sorted"), delta=kind == "delta"))
        try:
            _put(store, table, buf, True, keep)
            h2d[kind] = stats_of(store, table, filt, [], [lp.Count(T)])["h2d_bytes"]
            assert agg(db, table, filt, [], [lp.Count(T)]) == {(): (n - 200,)}
        finally:
            store.engine.drop_table(table)
            db.tables.pop(table, None)
    assert 0 < h2d["delta"] < h2d["twin"] / 4, h2d


@pytest.mark.parametrize("case", ["bit_width", "miniblock_overrun", "count"])
def test_corrupted_chunk_fails_only_the_queries_that_touch_it(store, case):
    name, buf, message = next(c for c in di.corrupted() if c[0] == case)
    db = store.DB(None, "delta_int64")
    keep = []
    for borrow in (False, True):
        table = f"dbp_corrupt_{case}_{int(borrow)}"
        _fresh(store, db, table, two_columns())
        try:
            _put(store, table, buf, borrow, keep)
            assert agg(db, table, None, [], [lp.Count(T), lp.Sum(T)]) == {(): (302, sum(range(302)))}
            with pytest.raises(_lib.FrostGPUError, match=re.escape("column value: " + message)) as e:
                agg(db, table, None, [], [lp.Sum(V)])
            assert e.value.code == _lib.FGPU_ERR_UNSUPPORTED
            with pytest.raises(_lib.FrostGPUError, match=re.escape(message)):
                agg(db, table, V.Gt(lp.Literal(0)), [], [lp.Count(T)])
        finally:
            store.engine.drop_table(table)
            db.tables.pop(table, None)
