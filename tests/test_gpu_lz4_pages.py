"""LZ4_RAW-compressed column chunks on the device (k_lz4_pages in lz4_pages.cu for PLAIN INT64 / DOUBLE value pages, the
host's inflation for everything else): every layout of tests/lz4_pages.py is put eagerly and borrowed, next to its
uncompressed twin and the same rows as an Arrow part, and then
- decode_column equals pyarrow's read, for every hand-assembled block too;
- Sum / Count / Min / Max by labels.a, labels.b under timestamp ranges, the numeric-edge literals and an OR filter, and
  filter-only plans, equal the twin's and numeric_edges' reference on every scan path, and the steady Execute takes the
  twin's kernels (fgpu_stats);
- compressed string layouts decode like pyarrow and dict_export lists the twin's order;
- the reference's filter_contains golden runs on parts with its `bytes` layout (`value` LZ4_RAW);
- a table mixing LZ4_RAW, uncompressed, DELTA_BINARY_PACKED and Arrow parts;
- the first Execute over a borrowed LZ4_RAW sorted part copies fewer bytes than the twin's, by what the footers save;
- a corrupted block fails only the queries that read its column, with its message."""
import os
import re

import numpy as np
import pyarrow as pa
import pytest

from frostdb_b200 import _lib
from frostdb_b200 import dynparquet as dp
from frostdb_b200 import logicalplan as lp
from frostdb_b200 import query
from tests import delta_int64 as di
from tests import golden_runner as gr
from tests import lz4_pages as lz
from tests import numeric_edges as ne
from tests import plain_strings as ps
from tests.golden.logictest_cases import CASES
from tests.test_gpu_delta_int64 import AGGS, PATHS, T, V, agg, edge_filters, or_filter, route, two_columns
from tests.test_gpu_plain_strings import SWITCHES, stats_of

pytestmark = pytest.mark.gpu

KINDS = ["eager", "borrow", "twin", "arrow"]


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


def _drop(store, db, tables):
    for t in tables:
        store.engine.drop_table(t)
        db.tables.pop(t, None)


def record_of(buf: bytes) -> pa.RecordBatch:
    """A part's rows as an Arrow record (dictionary labels as binary strings)."""
    t = dp.read_part(buf).combine_chunks()
    cols = []
    for n in t.schema.names:
        c = t.column(n).chunk(0)
        if pa.types.is_dictionary(c.type):
            c = c.cast(pa.string())
        if pa.types.is_string(c.type):
            c = c.cast(pa.binary())
        cols.append(c)
    return pa.RecordBatch.from_arrays(cols, names=t.schema.names)


@pytest.fixture(scope="module")
def parts(store):
    """Every layout as four tables of one part each: the LZ4_RAW file put eagerly and borrowed, the twin, the Arrow record."""
    db = store.DB(None, "lz4_pages")
    keep, made = [], {}
    for name in lz.NAMES:
        for kind in KINDS:
            table = f"lz4_{name}_{kind}"
            _fresh(store, db, table, lz.schema(name, lz4=kind != "twin"))
            if kind == "arrow":
                store.engine.put_arrow(table, record_of(lz.twin_of(name)))
            else:
                _put(store, table, lz.twin_of(name) if kind == "twin" else lz.file_of(name), kind == "borrow", keep)
            made[(name, kind)] = table
    yield db, made
    _drop(store, db, made.values())


def ts_filters(name):
    rg, n = lz.LAYOUT_BY_NAME[name].rg, len(lz.columns(name)["timestamp"])
    return [lp.And(T.GtEq(lp.Literal(rg // 2)), T.Lt(lp.Literal(rg + rg // 2))),
            lp.And(T.GtEq(lp.Literal(0)), T.Lt(lp.Literal(n))),
            T.GtEq(lp.Literal(n + 10))]


@pytest.mark.parametrize("kind", ["eager", "borrow"])
@pytest.mark.parametrize("name", lz.NAMES)
def test_decode_column_matches_pyarrow(store, parts, name, kind):
    _, made = parts
    t = dp.read_part(lz.twin_of(name))
    for col in ("timestamp", "value"):
        assert store.engine.decode_column(made[(name, kind)], 0, col).to_pylist() == t.column(col).to_pylist(), (name, kind, col)


@pytest.mark.parametrize("borrow", [False, True])
def test_hand_assembled_pages(store, borrow):
    """Every hand-assembled block as a v1 and a v2 page (literal and match lengths, offsets 1 .. 65 535, matches of
    matches, a 1 MiB run), a v2 page stored uncompressed, empty values regions and a compressed dictionary page."""
    db = store.DB(None, "lz4_pages")
    keep = []
    sch = two_columns()
    for c in sch.columns:
        c.delta_binary_packed = False
    for name, buf, exp, _ in lz.hand_layouts():
        table = f"lz4_hand_{name}_{int(borrow)}"
        _fresh(store, db, table, sch)
        try:
            _put(store, table, buf, borrow, keep)
            assert store.engine.decode_column(table, 0, "value").to_pylist() == exp, name
            aggs = [lp.Sum(V), lp.Count(V), lp.Min(V), lp.Max(V)]
            s = (sum(exp) + (1 << 63)) % (1 << 64) - (1 << 63)
            assert agg(db, table, None, [], aggs) == {(): (s, len(exp), min(exp), max(exp))}, name
        finally:
            _drop(store, db, [table])


@pytest.mark.parametrize("name", lz.NAMES)
def test_aggregates_equal_the_twin_and_the_reference(store, parts, name):
    db, made = parts
    phys = [ne.physical(lz.columns(name))]
    for filt in [None] + ts_filters(name) + [or_filter()]:
        exp = ne.reference(phys, filt, ne.KEYS, AGGS)
        what = f"{name} {filt.Name() if filt is not None else None}"
        for sw in PATHS:
            for kind in KINDS:
                ne.assert_same_result(agg(db, made[(name, kind)], filt, ne.KEYS, AGGS, sw), exp, AGGS, f"{what} {kind} {sw}")
            for kind in ("eager", "borrow"):
                assert route(store, made[(name, kind)], filt, ne.KEYS, AGGS, sw) == route(store, made[(name, "twin")], filt, ne.KEYS, AGGS, sw), \
                    f"{what} {kind} {sw}"
    for filt in edge_filters():
        exp = ne.reference(phys, filt, ne.KEYS, AGGS)
        for kind in KINDS:
            ne.assert_same_result(agg(db, made[(name, kind)], filt, ne.KEYS, AGGS), exp, AGGS, f"{name} {filt.Name()} {kind}")


@pytest.mark.parametrize("name", lz.NAMES)
def test_filter_only_plans(store, parts, name):
    db, made = parts
    phys = ne.physical(lz.columns(name))
    valid = phys.get("value#valid")
    names = ["timestamp", "value"]
    for filt in ts_filters(name)[:1] + [or_filter(), ne.leaf(ne.V, lp.OpGt, 0)]:
        sel = np.flatnonzero(ne.selection(phys, filt))
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


@pytest.mark.parametrize("name", lz.STR_NAMES)
def test_string_layouts(store, name):
    """decode_column of every column equals pyarrow's read, and dict_export after the compressed part equals the twin's."""
    db = store.DB(None, "lz4_pages")
    keep, tables = [], {}
    t = lz.str_table(name)
    try:
        for kind, buf in (("lz4", lz.str_file_of(name)), ("twin", lz.str_twin_of(name)), ("borrow", lz.str_file_of(name))):
            table = f"lz4_str_{name}_{kind}"
            _fresh(store, db, table, lz.str_schema() if kind != "twin" else ps.schema())
            _put(store, table, buf, kind == "borrow", keep)
            tables[kind] = table
            for col in ("s", "fvalue", "value"):
                exp = t.column(col).to_pylist()
                if col == "s":
                    exp = [None if v is None else v.encode() for v in exp]
                assert store.engine.decode_column(table, 0, col).to_pylist() == exp, (kind, col)
        for kind in ("lz4", "borrow"):
            assert store.engine.dict_export(tables[kind], "s") == store.engine.dict_export(tables["twin"], "s"), kind
    finally:
        _drop(store, db, tables.values())


def test_filter_contains_golden_on_lz4_parts(store, monkeypatch):
    """The reference's exec/filter/filter_contains on its `bytes` schema, `value` LZ4_RAW as upstream stores it."""
    case = next(c for c in CASES if c["source"].endswith("/filter_contains"))
    monkeypatch.setitem(gr.SCHEMAS, "bytes", lambda: lz.bytes_schema(True))
    db = store.DB(None, "lz4_pages")
    name = "lz4_golden_filter_contains"
    if name in db.tables:
        _drop(store, db, [name])
    ran = 0
    try:
        for ex, got, exp in gr.run_case(case, lambda s: db.Table(name, s),
                                        lambda: query.NewEngine(None, db.TableProvider()).ScanTable(name),
                                        supports=lambda k: k in {"aggregate", "distinct", "filter"}):
            gr.check(ex, got, exp)
            ran += 1
    finally:
        _drop(store, db, [name])
    assert ran > 0


def test_mixed_table(store):
    """An LZ4_RAW, an uncompressed, a DELTA_BINARY_PACKED and an Arrow part give what four uncompressed parts give."""
    db = store.DB(None, "lz4_pages")
    names = ["sorted", "unsorted", "delta", "page_edges"]
    mixed, plain, keep = "lz4_table_mixed", "lz4_table_plain", []
    try:
        _fresh(store, db, mixed, lz.schema("sorted", lz4=True))
        _put(store, mixed, lz.file_of(names[0]), False, keep)
        _put(store, mixed, lz.twin_of(names[1]), True, keep)
        _put(store, mixed, di.file_of("sorted"), False, keep)
        store.engine.put_arrow(mixed, record_of(lz.twin_of(names[3])))
        _fresh(store, db, plain, lz.schema("sorted", lz4=False))
        for buf in (lz.twin_of(names[0]), lz.twin_of(names[1]), di.twin_of("sorted"), lz.twin_of(names[3])):
            _put(store, plain, buf, False, keep)
        phys = [ne.physical(lz.columns(names[0])), ne.physical(lz.columns(names[1])), ne.physical(di.columns("sorted")),
                ne.physical(lz.columns(names[3]))]
        for filt in [None, or_filter()] + ts_filters("sorted")[:1]:
            exp = ne.reference(phys, filt, ne.KEYS, AGGS)
            ne.assert_same_result(agg(db, mixed, filt, ne.KEYS, AGGS), exp, AGGS, "mixed")
            ne.assert_same_result(agg(db, plain, filt, ne.KEYS, AGGS), exp, AGGS, "plain")
    finally:
        _drop(store, db, [mixed, plain])


def test_first_execute_of_a_borrowed_sorted_part_copies_what_the_footers_save(store):
    """`timestamp` and `value` of a sorted part: the LZ4_RAW part's first Execute copies the twin's bytes less what
    compression saves on the two columns (the blocks replace the values; the directories and tables are the same)."""
    db = store.DB(None, "lz4_pages")
    keep, h2d = [], {}
    n = len(lz.columns("sorted")["timestamp"])
    filt = lp.And(T.GtEq(lp.Literal(100)), T.Lt(lp.Literal(n - 100)))
    aggs = [lp.Sum(V), lp.Count(T)]
    for kind, buf in (("lz4", lz.file_of("sorted")), ("twin", lz.twin_of("sorted"))):
        table = f"lz4_h2d_{kind}"
        _fresh(store, db, table, lz.schema("sorted", lz4=kind == "lz4"))
        try:
            _put(store, table, buf, True, keep)
            h2d[kind] = stats_of(store, table, filt, [], aggs)["h2d_bytes"]
        finally:
            _drop(store, db, [table])
    saved = sum(lz.footer_sizes(lz.file_of("sorted"), c)[1] - lz.footer_sizes(lz.file_of("sorted"), c)[0] for c in ("timestamp", "value"))
    assert saved > 0
    assert h2d["lz4"] < h2d["twin"], h2d
    # (each page adds a job to the table and its block's padding; the page headers the twin's coalesced copies carry are gone)
    assert abs((h2d["twin"] - h2d["lz4"]) - saved) < 0.05 * saved + 64 * 1024, (h2d, saved)


@pytest.mark.parametrize("case", ["offset_0", "offset_past_output", "output_longer", "trailing_bytes"])
def test_corrupted_block_fails_only_the_queries_that_read_its_column(store, case):
    name, buf, message = next(c for c in lz.corrupted_files() if c[0] == case)
    db = store.DB(None, "lz4_pages")
    keep = []
    n = _lib.describe_parquet(buf)["row_groups"][0]["n_rows"]
    for borrow in (False, True):
        table = f"lz4_corrupt_{case}_{int(borrow)}"
        _fresh(store, db, table, two_columns())
        try:
            _put(store, table, buf, borrow, keep)
            assert agg(db, table, None, [], [lp.Count(T), lp.Sum(T)]) == {(): (n, sum(range(n)))}
            with pytest.raises(_lib.FrostGPUError, match=re.escape("column value: " + message)) as e:
                agg(db, table, None, [], [lp.Sum(V)])
            assert e.value.code == _lib.FGPU_ERR_UNSUPPORTED
            with pytest.raises(_lib.FrostGPUError, match=re.escape(message)):
                agg(db, table, V.Gt(lp.Literal(0)), [], [lp.Count(T)])
        finally:
            _drop(store, db, [table])
