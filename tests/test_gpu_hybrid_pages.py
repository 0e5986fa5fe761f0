"""The device half of the hybrid-stream decoder on the layout zoo of tests/hybrid_pages.py, against pyarrow's read:
every file is put eagerly and borrowed, and then
- decode_column (k_decode, HybCur, the device seeds) equals pyarrow's read for every column;
- aggregate plans over the zoo columns (k_runs_tma on row-space directories, k_tile_agg on k_flatten's codes, fast_pass,
  k_scan) equal the numpy reference exactly under every switch set, and with the default switches the sorted layouts
  take the sorted-run kernel and the bit-packed ones the tile kernel;
- filter-only plans (k_take_*, k_rows) return pyarrow's rows in order;
- the over-wide chunks are refused with FrostGPUError."""
import ctypes as C
import os

import numpy as np
import pyarrow as pa
import pytest

from frostdb_b200 import _lib
from frostdb_b200 import logicalplan as lp
from frostdb_b200 import query
from frostdb_b200.physicalplan import GPUScan
from tests import hybrid_pages as hp
from tests import numeric_edges as ne

pytestmark = pytest.mark.gpu

AGG_SWITCHES = [{}, {"FROSTGPU_NO_RUNS": "1"}, {"FROSTGPU_NO_RUNS": "1", "FROSTGPU_NO_TILE": "1"},
                {"FROSTGPU_NO_RUNS": "1", "FROSTGPU_NO_TILE": "1", "FROSTGPU_NO_FAST": "1"}, {"FROSTGPU_NO_PRUNE": "1"}]
ALL_SWITCHES = ("FROSTGPU_NO_RUNS", "FROSTGPU_NO_TILE", "FROSTGPU_NO_FAST", "FROSTGPU_NO_PRUNE", "FROSTGPU_NO_TAKE")
NAMES = [l.name for l in hp.LAYOUTS]
MODES = ["eager", "borrow"]


@pytest.fixture(autouse=True)
def clean_switches():
    yield
    for k in ALL_SWITCHES:
        os.environ.pop(k, None)


@pytest.fixture(scope="module")
def zoo(store):
    """Every zoo file as a table of its own, put eagerly and borrowed (from caller-owned memory)."""
    db = store.DB(None, "hybrid_pages")
    keep, made = [], {}
    for name in NAMES:
        buf = hp.file_of(name)
        for mode in MODES:
            table = f"hybrid_{name}_{mode}"
            if table in db.tables:
                store.engine.drop_table(table)
            db.Table(table, hp.schema())
            if mode == "borrow":
                arr = np.frombuffer(buf, dtype=np.uint8)
                keep.append(arr)
                store.engine.put_parquet(table, arr, borrow=True)
            else:
                store.engine.put_parquet(table, buf)
            made[(name, mode)] = table
    yield db, made
    for table in made.values():
        store.engine.drop_table(table)
        db.tables.pop(table, None)


@pytest.fixture(scope="module")
def refs():
    return {}


def reference(refs, name):
    if name not in refs:
        refs[name] = hp.Reference(name)
    return refs[name]


def run_agg(db, table, filt, keys, aggs):
    out = []
    q = query.NewEngine(None, db.TableProvider()).ScanTable(table)
    q = q.Filter(filt) if filt is not None else q
    q.Aggregate(aggs, [lp.Col(k) for k in keys]).Execute(None, lambda c, r: out.append(r))
    return ne.result_map(out, keys, aggs)


def stats_of(store, table, filt, keys, aggs):
    eng, lib = store.engine, _lib.load()
    q, keep = GPUScan(eng, table, filt, _lib.PLAN_AGGREGATE, [lp.Col(k) for k in keys], aggs).prepare()
    res = C.c_void_p()
    try:
        _lib.check(lib.fgpu_query_execute(eng.handle, q, eng.table_watermark(table), C.byref(res)))
        st = eng.stats(res)
        lib.fgpu_result_free(res)
    finally:
        lib.fgpu_query_free(q)
    return st


def with_switches(sw, fn):
    os.environ.update(sw)
    try:
        return fn()
    finally:
        for k in sw:
            os.environ.pop(k)


def plain(a) -> pa.Array:
    """An engine column as pyarrow reads the file: dictionaries decoded, byte strings as UTF-8."""
    if isinstance(a, pa.ChunkedArray):
        a = pa.concat_arrays(a.chunks) if a.num_chunks else pa.array([], pa.int64())
    if pa.types.is_dictionary(a.type):
        a = a.dictionary_decode()
    return a.cast(pa.string()) if pa.types.is_binary(a.type) or pa.types.is_large_binary(a.type) else a


def assert_same_array(got: pa.Array, exp: pa.Array, what: str) -> None:
    assert len(got) == len(exp), f"{what}: {len(got)} rows, expected {len(exp)}"
    if not got.equals(exp):
        g, e = got.to_pylist(), exp.to_pylist()
        i = next(i for i, (x, y) in enumerate(zip(g, e)) if x != y)
        raise AssertionError(f"{what}: row {i}: got {g[i]!r}, expected {e[i]!r}")


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", NAMES)
def test_decode_column_matches_pyarrow(store, zoo, name, mode):
    layout = hp.LAYOUT_BY_NAME[name]
    _, made = zoo
    t = hp.read(name)
    for col in t.column_names:
        if layout.error and col in ("labels.z", "dictvalue"):
            with pytest.raises(_lib.FrostGPUError, match=layout.error):
                store.engine.decode_column(made[(name, mode)], 0, col)
            continue
        assert_same_array(plain(store.engine.decode_column(made[(name, mode)], 0, col)), plain(t.column(col)), f"{name} {mode} {col}")


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", [l.name for l in hp.LAYOUTS if not l.error])
def test_aggregates_match_the_reference(store, zoo, refs, name, mode):
    layout = hp.LAYOUT_BY_NAME[name]
    db, made = zoo
    table, ref = made[(name, mode)], reference(refs, name)
    for filt, keys, aggs in hp.plans(layout):
        exp = ref.aggregate(filt, keys, aggs)
        for sw in AGG_SWITCHES:
            got = with_switches(sw, lambda: run_agg(db, table, filt, keys, aggs))
            ne.assert_same_result(got, exp, aggs, f"{table} filter {filt.Name() if filt is not None else None} {keys} {sw}")


@pytest.mark.parametrize("name", [l.name for l in hp.LAYOUTS if not l.error])
def test_kernel_that_takes_the_row_groups(store, zoo, name):
    """Sorted layouts (nullable run-length ones included) on k_runs_tma, bit-packed ones on k_tile_agg: every row group,
    keyed by one and by two zoo columns, without a filter, with a timestamp range that prunes nothing away, and with
    a dictionary leaf on labels.z (the sorted-run kernel walks the leaf's row-space directory, the tile kernel reads
    its flat codes)."""
    layout = hp.LAYOUT_BY_NAME[name]
    _, made = zoo
    aggs = [lp.Sum(lp.Col("value")), lp.Count(lp.Col("value")), lp.Min(lp.Col("value")), lp.Max(lp.Col("value"))]
    n = sum(layout.rg_rows)
    z_leaf = lp.Col("labels.z").Eq(lp.Literal(hp.zoo_literal(layout)))
    for filt in (None, lp.Col("timestamp").GtEq(lp.Literal(0)), lp.Col("timestamp").Lt(lp.Literal(n)), z_leaf):
        for keys in (["labels.z"], ["labels.z", "labels.y"]):
            st = stats_of(store, made[(name, "eager")], filt, keys, aggs)
            kernel = "row_groups_runs" if layout.sorted else "row_groups_tiles"
            assert st["row_groups"] == len(layout.rg_rows) and st[kernel] == st["row_groups"], (keys, filt.Name() if filt else None, st)


@pytest.mark.parametrize("name", [l.name for l in hp.LAYOUTS if l.error])
def test_over_wide_chunks_are_refused(zoo, name):
    db, made = zoo
    for mode in MODES:
        for keys, aggs in ((["labels.z"], [lp.Sum(lp.Col("value"))]), (["labels.y"], [lp.Sum(lp.Col("dictvalue"))])):
            with pytest.raises(_lib.FrostGPUError, match=hp.LAYOUT_BY_NAME[name].error):
                run_agg(db, made[(name, mode)], None, keys, aggs)
    # the other columns of the file still answer
    ref = hp.Reference(name)
    aggs = [lp.Sum(lp.Col("value")), lp.Count(lp.Col("value"))]
    ne.assert_same_result(run_agg(db, made[(name, "eager")], None, ["labels.y"], aggs), ref.aggregate(None, ["labels.y"], aggs), aggs)


def check_rows(db, table, ref, filt, names, what):
    out = []
    query.NewEngine(None, db.TableProvider()).ScanTable(table).Filter(filt).Project(*[lp.Col(c) for c in names]) \
        .Execute(None, lambda c, r: out.append(r))
    exp = ref.rows(filt, names)
    batches = [b for b in out if b.num_rows]  # (empty records carry no columns)
    for c in names:
        got = [plain(b.column(b.schema.get_field_index(c))) for b in batches]
        got = pa.concat_arrays(got) if got else exp[c][:0]
        assert_same_array(got, exp[c], f"{what} {c}")
    return len(exp[names[0]])


def rows_plan_launches(store, table, filt, names):
    eng, lib = store.engine, _lib.load()
    q, keep = GPUScan(eng, table, filt, _lib.PLAN_FILTER, [lp.Col(c) for c in names], []).prepare()
    res = C.c_void_p()
    try:
        _lib.check(lib.fgpu_query_execute(eng.handle, q, eng.table_watermark(table), C.byref(res)))
        st = eng.stats(res)
        lib.fgpu_result_free(res)
    finally:
        lib.fgpu_query_free(q)
    return st["kernel_launches"]


@pytest.mark.parametrize("name", [l.name for l in hp.LAYOUTS if not l.error])
def test_filter_only_rows_on_the_take_kernels_and_k_rows(store, zoo, refs, name):
    """Leaves on labels.z (evaluated on k_flatten's flat codes) and timestamp, projecting PLAIN columns: the ordered
    take kernels by default, k_rows with FROSTGPU_NO_TAKE, both returning pyarrow's rows in order.  The take path
    launches its two kernels (count, then gather) where k_rows is one launch."""
    layout = hp.LAYOUT_BY_NAME[name]
    db, made = zoo
    ref, table, names = reference(refs, name), made[(name, "eager")], ["timestamp", "value"]
    for filt in hp.zoo_filters(layout):
        for sw in ({}, {"FROSTGPU_NO_TAKE": "1"}):
            n = with_switches(sw, lambda: check_rows(db, table, ref, filt, names, f"{name} {filt.Name()} {sw}"))
        take = rows_plan_launches(store, table, filt, names)
        rows = with_switches({"FROSTGPU_NO_TAKE": "1"}, lambda: rows_plan_launches(store, table, filt, names))
        # (`== NULL` on a REQUIRED column: the null counts prune every row group and nothing is launched)
        assert take == rows + 2 or take == rows == n == 0, \
            f"{name} {filt.Name()}: {take} launches with the take kernels, {rows} on k_rows, {n} rows"


@pytest.mark.parametrize("name", [l.name for l in hp.LAYOUTS if not l.error])
def test_filter_only_rows_with_dictionary_outputs(zoo, refs, name):
    """Projecting labels.z and the nullable dictvalue: k_rows decodes both through HybCur.  Besides the aggregate plans'
    filters, a general filter program with two leaves on dictvalue."""
    layout = hp.LAYOUT_BY_NAME[name]
    db, made = zoo
    ref = reference(refs, name)
    filters = {f.Name(): f for f, _, _ in hp.plans(layout) if f is not None}
    dv, z = lp.Col("dictvalue"), lp.Col("labels.z")
    program = lp.And(lp.Or(dv.Lt(lp.Literal(2)), dv.Gt(lp.Literal(5))), z.NotEq(lp.Literal(hp.zoo_literal(layout))))
    filters[program.Name()] = program
    for filt in filters.values():
        check_rows(db, made[(name, "eager")], ref, filt, ["labels.z", "value", "dictvalue"], f"{name} {filt.Name()}")
