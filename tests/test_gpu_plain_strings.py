"""PLAIN string column chunks on the device (intern_strings.cu): every layout of tests/plain_strings.py is put eagerly
and borrowed, next to its RLE_DICTIONARY twin and the same rows as an Arrow part, and then
- decode_column equals pyarrow's read, and dict_export lists what the Arrow part's host interning lists;
- a PLAIN, a dictionary and an Arrow part in one table share their global ids;
- group-by on `s`, leaves on it (==, !=, regex, contains, == NULL), an OR filter, Distinct and filter-only plans give
  the twin's and pyarrow's answers, on the kernels named through fgpu_stats;
- values with equal first bytes and different lengths, and many distinct values in one chunk, each get their own id."""
import ctypes as C
import math
import os
import re

import pyarrow as pa
import pyarrow.compute as pc
import pytest

from frostdb_b200 import _lib
from frostdb_b200 import logicalplan as lp
from frostdb_b200 import query
from frostdb_b200.physicalplan import GPUScan
from tests import plain_strings as ps

pytestmark = pytest.mark.gpu

SWITCHES = ("FROSTGPU_NO_RUNS", "FROSTGPU_NO_TILE", "FROSTGPU_NO_FAST", "FROSTGPU_NO_PRUNE", "FROSTGPU_NO_TAKE")
KINDS = ["eager", "borrow", "twin", "arrow"]
V, F, S = lp.Col("value"), lp.Col("fvalue"), lp.Col("s")
AGGS = [lp.Sum(V), lp.Count(V), lp.Min(V), lp.Max(V), lp.Sum(F)]


@pytest.fixture(autouse=True)
def clean_switches():
    yield
    for k in SWITCHES:
        os.environ.pop(k, None)


@pytest.fixture(scope="module")
def parts(store):
    """Every layout as four tables of one part each: PLAIN put eagerly, PLAIN borrowed, the twin, the Arrow record."""
    import numpy as np
    db = store.DB(None, "plain_strings")
    keep, made = [], {}
    for name in ps.NAMES:
        for kind in KINDS:
            table = f"plain_{name}_{kind}"
            if table in db.tables:
                store.engine.drop_table(table)
            db.Table(table, ps.schema())
            if kind == "borrow":
                arr = np.frombuffer(ps.file_of(name), dtype=np.uint8)
                keep.append(arr)
                store.engine.put_parquet(table, arr, borrow=True)
            elif kind == "arrow":
                store.engine.put_arrow(table, ps.record_of(name))
            else:
                store.engine.put_parquet(table, ps.twin_of(name) if kind == "twin" else ps.file_of(name))
            made[(name, kind)] = table
    yield db, made
    for table in made.values():
        store.engine.drop_table(table)
        db.tables.pop(table, None)


def as_strings(a) -> list:
    if isinstance(a, pa.ChunkedArray):
        a = pa.concat_arrays(a.chunks)
    if pa.types.is_dictionary(a.type):
        a = a.dictionary_decode()
    return [x.decode() if isinstance(x, bytes) else x for x in a.to_pylist()]


def run(db, table, build):
    out = []
    build(query.NewEngine(None, db.TableProvider()).ScanTable(table)).Execute(None, lambda c, r: out.append(r))
    return [b for b in out if b.num_rows]


def groups(batches, keys, aggs) -> dict:
    names = list(keys) + [a.Name() for a in aggs]
    out = {}
    for b in batches:
        cols = [as_strings(b.column(b.schema.get_field_index(n))) for n in names]
        for r in zip(*cols):
            assert r[: len(keys)] not in out, r
            out[r[: len(keys)]] = r[len(keys):]
    return out


def same(got, exp, what):
    """Keys, counts and int64 aggregates exactly; float sums within 1e-9 relative (another kernel adds in another order)."""
    assert set(got) == set(exp), f"{what}: groups differ: {sorted(set(got) ^ set(exp), key=str)[:5]}"
    for k, ev in exp.items():
        for g, e in zip(got[k], ev):
            if e is None:  # Sum(fvalue) of a group whose fvalue is NULL throughout
                assert g is None or g == 0.0, f"{what}: {k}: {g!r} vs {e!r}"
            elif isinstance(e, float) or isinstance(g, float):
                assert math.isclose(g, e, rel_tol=1e-9, abs_tol=1e-9), f"{what}: {k}: {g!r} vs {e!r}"
            else:
                assert g == e, f"{what}: {k}: {g!r} vs {e!r}"


def reference(name, mask_of, keys) -> dict:
    """pyarrow: Sum / Count / Min / Max of value and Sum of fvalue per key over the rows the mask selects."""
    t = ps.table(name)
    cols = {n: t.column(n).to_pylist() for n in t.column_names}
    out = {}
    for i in range(t.num_rows):
        if not mask_of(cols, i):
            continue
        k = tuple(cols[c][i] for c in keys)
        acc = out.setdefault(k, [0, 0, None, None, None])
        v, f = cols["value"][i], cols["fvalue"][i]
        acc[0] += v
        acc[1] += 1
        acc[2] = v if acc[2] is None else min(acc[2], v)
        acc[3] = v if acc[3] is None else max(acc[3], v)
        if f is not None:
            acc[4] = f if acc[4] is None else acc[4] + f
    return {k: tuple(v) for k, v in out.items()}


def literal(name) -> str:
    """A frequent value of `s`."""
    vals = [v for v in ps.table(name).column("s").to_pylist() if v is not None]
    return max(set(vals), key=vals.count) if vals else "absent"


def filters(name):
    """(filter, row predicate) pairs: leaves on `s`, and an OR that only the general scan kernel takes."""
    lit = literal(name)
    sub = lit[1:3] if len(lit) >= 3 else lit
    rx = "^" + re.escape(lit[:2]) if lit else "^$"
    return [
        (S.Eq(lp.Literal(lit)), lambda c, i: c["s"][i] == lit),
        (S.NotEq(lp.Literal(lit)), lambda c, i: c["s"][i] is not None and c["s"][i] != lit),
        (S.RegexMatch(rx), lambda c, i: c["s"][i] is not None and re.search(rx, c["s"][i]) is not None),
        (S.Contains(sub), lambda c, i: c["s"][i] is not None and sub in c["s"][i]),
        (S.Eq(lp.Literal(None)), lambda c, i: c["s"][i] is None),
        (lp.Or(S.Eq(lp.Literal(lit)), V.Lt(lp.Literal(-900))), lambda c, i: c["s"][i] == lit or c["value"][i] < -900),
    ]


def stats_of(store, table, filt, keys, aggs, kind=_lib.PLAN_AGGREGATE):
    eng, lib = store.engine, _lib.load()
    q, keep = GPUScan(eng, table, filt, kind, [lp.Col(k) for k in keys], aggs).prepare()
    res = C.c_void_p()
    try:
        _lib.check(lib.fgpu_query_execute(eng.handle, q, eng.table_watermark(table), C.byref(res)))
        st = eng.stats(res)
        lib.fgpu_result_free(res)
    finally:
        lib.fgpu_query_free(q)
    return st


@pytest.mark.parametrize("kind", ["eager", "borrow"])
@pytest.mark.parametrize("name", ps.NAMES)
def test_decode_column_matches_pyarrow(store, parts, name, kind):
    _, made = parts
    t = ps.table(name)
    for col in t.column_names:
        got = store.engine.decode_column(made[(name, kind)], 0, col)
        exp = t.column(col).to_pylist()
        assert (as_strings(got) if col == "s" else got.to_pylist()) == exp, (name, kind, col)


@pytest.mark.parametrize("name", ps.NAMES)
def test_dict_export_equals_the_arrow_parts(store, parts, name):
    _, made = parts
    exp = store.engine.dict_export(made[(name, "arrow")], "s")
    assert exp == [v.encode() for v in ps.first_occurrence(ps.table(name).column("s").to_pylist())]
    for kind in ("eager", "borrow"):
        store.engine.decode_column(made[(name, kind)], 0, "s")  # a borrowed part interns when the column is first needed
        assert store.engine.dict_export(made[(name, kind)], "s") == exp, kind


@pytest.mark.parametrize("name", ["fallback_v2", "v1_optional", "collisions"])
def test_plain_dictionary_and_arrow_parts_share_ids(store, name):
    """Three parts with the same rows: every group counts three times its rows, and the dictionary is the one list."""
    db = store.DB(None, "plain_strings")
    table = f"plain_shared_{name}"
    if table in db.tables:
        store.engine.drop_table(table)
    db.Table(table, ps.schema())
    try:
        store.engine.put_parquet(table, ps.file_of(name))
        store.engine.put_parquet(table, ps.twin_of(name))
        store.engine.put_arrow(table, ps.record_of(name))
        got = groups(run(db, table, lambda q: q.Aggregate([lp.Count(V), lp.Sum(V)], [S])), ["s"], [lp.Count(V), lp.Sum(V)])
        exp = {k: (3 * v[1], 3 * v[0]) for k, v in reference(name, lambda c, i: True, ["s"]).items()}
        same(got, exp, name)
        assert store.engine.dict_export(table, "s") == [v.encode() for v in ps.first_occurrence(ps.table(name).column("s").to_pylist())]
    finally:
        store.engine.drop_table(table)
        db.tables.pop(table, None)


@pytest.mark.parametrize("name", ps.NAMES)
def test_group_by_and_leaves_match_the_twin_and_pyarrow(store, parts, name):
    db, made = parts
    plans = [(None, lambda c, i: True)] + filters(name)
    for filt, pred in plans:
        build = (lambda q: q.Filter(filt).Aggregate(AGGS, [S])) if filt is not None else (lambda q: q.Aggregate(AGGS, [S]))
        exp = reference(name, pred, ["s"])
        what = f"{name} {filt.Name() if filt is not None else None}"
        twin = groups(run(db, made[(name, "twin")], build), ["s"], AGGS)
        same(twin, exp, what + " twin")
        for kind in ("eager", "borrow", "arrow"):
            same(groups(run(db, made[(name, kind)], build), ["s"], AGGS), exp, f"{what} {kind}")
        # the same leaves without a key: `s` only in the filter
        build2 = (lambda q: q.Filter(filt).Aggregate([lp.Count(V)], [])) if filt is not None else (lambda q: q.Aggregate([lp.Count(V)], []))
        n = sum(v[1] for v in exp.values())
        got = groups(run(db, made[(name, "eager")], build2), [], [lp.Count(V)])
        assert got.get((), (0,))[0] == n, what


@pytest.mark.parametrize("name", ["v2_optional", "fallback_v1", "collisions", "many_small_pages"])
def test_kernels_that_take_the_row_groups(store, parts, name):
    """Group-by on `s` and a leaf on it: the tile kernel (k_flatten's codes); an OR filter: the general kernel.  The
    twin's row groups go the same way."""
    _, made = parts
    table = made[(name, "eager")]
    n_rg = len(ps.row_group_slices(ps.file_of(name)))
    lit = literal(name)
    aggs = [lp.Sum(V), lp.Count(V), lp.Min(V), lp.Max(V)]  # (Sum of the nullable fvalue is the general kernel's)
    route = ("row_groups", "row_groups_tiles", "row_groups_runs")
    for filt in (None, S.Eq(lp.Literal(lit))):
        st = stats_of(store, table, filt, ["s"], aggs)
        assert st["row_groups"] == n_rg and st["row_groups_tiles"] == n_rg and st["row_groups_runs"] == 0, st
        tw = stats_of(store, made[(name, "twin")], filt, ["s"], aggs)
        assert [st[k] for k in route] == [tw[k] for k in route], (st, tw)
    st = stats_of(store, table, lp.Or(S.Eq(lp.Literal(lit)), V.Lt(lp.Literal(-900))), ["s"], aggs)
    assert st["row_groups"] == n_rg and st["row_groups_tiles"] == 0 and st["row_groups_runs"] == 0, st
    os.environ["FROSTGPU_NO_TILE"] = "1"
    st = stats_of(store, table, None, ["s"], AGGS)
    assert st["row_groups_tiles"] == 0 and st["row_groups_runs"] == 0, st
    same(groups(run(parts[0], table, lambda q: q.Aggregate(AGGS, [S])), ["s"], AGGS),
         reference(name, lambda c, i: True, ["s"]), f"{name} on k_scan")


@pytest.mark.parametrize("name", ps.NAMES)
def test_distinct_and_hash_keys(parts, name):
    db, made = parts
    exp = {(v,) for v in ps.table(name).column("s").to_pylist() if v is not None}
    seen = {}
    for kind in ("eager", "borrow", "twin"):
        got = []
        for b in run(db, made[(name, kind)], lambda q: q.Distinct(S)):
            got.extend((v,) for v in as_strings(b.column(b.schema.get_field_index("s"))))
        assert len(got) == len(set(got)), kind
        seen[kind] = set(got)
        assert seen[kind] - {(None,)} == exp, kind
    assert seen["eager"] == seen["borrow"] == seen["twin"]
    # (s, value): a key space the dense table cannot hold
    keys = [S, V]
    exp2 = reference(name, lambda c, i: True, ["s", "value"])
    got2 = groups(run(db, made[(name, "eager")], lambda q: q.Aggregate([lp.Count(V)], keys)), ["s", "value"], [lp.Count(V)])
    same(got2, {k: (v[1],) for k, v in exp2.items()}, f"{name} (s, value)")


def rows_of(db, table, filt, names):
    out = run(db, table, lambda q: q.Filter(filt).Project(*[lp.Col(n) for n in names]))
    rows = []
    for b in out:
        cols = [as_strings(b.column(b.schema.get_field_index(n))) for n in names]
        rows.extend(zip(*cols))
    return rows


def launches(store, table, filt, names):
    return stats_of(store, table, filt, names, [], kind=_lib.PLAN_FILTER)["kernel_launches"]


@pytest.mark.parametrize("name", ps.NAMES)
def test_filter_only_plans(store, parts, name):
    """Projecting `s` (k_rows decodes it through its directory) and a leaf on `s` projecting the numeric columns (the
    ordered take kernels: two launches more than k_rows)."""
    db, made = parts
    t = ps.table(name)
    cols = {n: t.column(n).to_pylist() for n in t.column_names}
    for filt, pred in filters(name):
        sel = [i for i in range(t.num_rows) if pred(cols, i)]
        for kind in ("eager", "borrow"):
            table = made[(name, kind)]
            got = rows_of(db, table, filt, ["timestamp", "s"])
            assert got == [(cols["timestamp"][i], cols["s"][i]) for i in sel], (name, kind, filt.Name())
            got = rows_of(db, table, filt, ["timestamp", "value"])
            assert got == [(cols["timestamp"][i], cols["value"][i]) for i in sel], (name, kind, filt.Name())
        if filt.Op == lp.OpOr:
            continue
        take = launches(store, made[(name, "eager")], filt, ["timestamp", "value"])
        os.environ["FROSTGPU_NO_TAKE"] = "1"
        rows = launches(store, made[(name, "eager")], filt, ["timestamp", "value"])
        os.environ.pop("FROSTGPU_NO_TAKE")
        assert take == rows + 2 or take == rows == len(sel) == 0, (name, filt.Name(), take, rows)


def test_every_distinct_string_gets_its_own_id(store, parts):
    """Equal first bytes, lengths 0 .. 299 (and xy-repeats), and 20 000 distinct values in one chunk."""
    _, made = parts
    s = ps.table("collisions").column("s").to_pylist()
    exp = ps.first_occurrence(s)
    assert len(exp) == ps.LAYOUT_BY_NAME["collisions"].n_distinct
    assert store.engine.dict_export(made[("collisions", "eager")], "s") == [v.encode() for v in exp]
    got = store.engine.decode_column(made[("collisions", "eager")], 0, "s")
    assert as_strings(got) == s
    ids = got.indices.to_pylist() if pa.types.is_dictionary(got.type) else None
    if ids is not None:
        by_value = {}
        for v, i in zip(s, ids):
            assert by_value.setdefault(v, i) == i, v
        assert len(set(by_value.values())) == len(by_value)
