"""DELTA_LENGTH_BYTE_ARRAY and DELTA_BYTE_ARRAY string column chunks on the device (k_str_unfront, k_str_hash,
k_str_gather in intern_strings.cu): every layout of tests/delta_strings.py is put eagerly and borrowed, next to its
RLE_DICTIONARY twin, its PLAIN twin and the same rows as an Arrow part, and then
- decode_column equals pyarrow's read, and dict_export lists what the Arrow part's and the PLAIN twin's list;
- a delta, a PLAIN, a dictionary and an Arrow part in one table share their global ids;
- group-by on `s`, leaves on it, an OR filter, Distinct, hash-table keys and filter-only plans give the twin's and
  pyarrow's answers, on the kernels fgpu_stats names for the twin;
- a chunk with a corrupted delta page fails the queries that touch its column only."""
import os
import re

import pyarrow as pa
import pytest

from frostdb_b200 import _lib
from frostdb_b200 import dynparquet as dp
from frostdb_b200 import logicalplan as lp
from tests import delta_strings as ds
from tests.test_gpu_plain_strings import AGGS, S, SWITCHES, V, as_strings, groups, launches, rows_of, run, same, stats_of

pytestmark = pytest.mark.gpu

KINDS = ["eager", "borrow", "twin", "plain", "arrow"]


@pytest.fixture(autouse=True)
def clean_switches():
    yield
    for k in SWITCHES:
        os.environ.pop(k, None)


def _fresh(store, db, table):
    if table in db.tables:
        store.engine.drop_table(table)
    db.Table(table, ds.schema())


@pytest.fixture(scope="module")
def parts(store):
    """Every case as five tables of one part each: the delta file put eagerly and borrowed, the RLE_DICTIONARY twin, the
    PLAIN twin, the Arrow record."""
    import numpy as np
    db = store.DB(None, "delta_strings")
    keep, made = [], {}
    for name, enc in ds.CASES:
        for kind in KINDS:
            table = f"delta_{name}_{enc}_{kind}"
            _fresh(store, db, table)
            if kind == "borrow":
                arr = np.frombuffer(ds.file_of(name, enc), dtype=np.uint8)
                keep.append(arr)
                store.engine.put_parquet(table, arr, borrow=True)
            elif kind == "arrow":
                store.engine.put_arrow(table, ds.record_of(name))
            else:
                buf = {"eager": ds.file_of(name, enc), "twin": ds.twin_of(name), "plain": ds.plain_of(name)}[kind]
                store.engine.put_parquet(table, buf)
            made[(name, enc, kind)] = table
    yield db, made
    for table in made.values():
        store.engine.drop_table(table)
        db.tables.pop(table, None)


def two_columns() -> dp.Schema:
    """The schema of the hand-assembled files: `s` and `timestamp`."""
    return dp.Schema(name="assembled", columns=[dp.ColumnDefinition("s", dp.TYPE_STRING), dp.ColumnDefinition("timestamp", dp.TYPE_INT64)],
                     sorting_columns=[dp.SortingColumn("timestamp")])


def reference(name, mask_of, keys) -> dict:
    t = ds.table(name)
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
    vals = [v for v in ds.table(name).column("s").to_pylist() if v is not None]
    return max(set(vals), key=vals.count) if vals else "absent"


def filters(name):
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


@pytest.mark.parametrize("kind", ["eager", "borrow"])
@pytest.mark.parametrize("name,enc", ds.CASES, ids=ds.CASE_IDS)
def test_decode_column_matches_pyarrow(store, parts, name, enc, kind):
    _, made = parts
    t = ds.table(name)
    for col in t.column_names:
        got = store.engine.decode_column(made[(name, enc, kind)], 0, col)
        exp = t.column(col).to_pylist()
        assert (as_strings(got) if col == "s" else got.to_pylist()) == exp, (name, enc, kind, col)


@pytest.mark.parametrize("name,enc", ds.CASES, ids=ds.CASE_IDS)
def test_dict_export_equals_the_arrow_parts_and_the_plain_twins(store, parts, name, enc):
    _, made = parts
    exp = store.engine.dict_export(made[(name, enc, "arrow")], "s")
    assert exp == [v.encode() for v in ds.first_occurrence(ds.table(name).column("s").to_pylist())]
    for kind in ("eager", "borrow", "plain"):
        store.engine.decode_column(made[(name, enc, kind)], 0, "s")  # a borrowed part interns when the column is first needed
        assert store.engine.dict_export(made[(name, enc, kind)], "s") == exp, kind


@pytest.mark.parametrize("name", ["v2_optional", "collisions", "sorted_prefixes", "long_chain"])
def test_delta_plain_dictionary_and_arrow_parts_share_ids(store, name):
    """Five parts with the same rows: every group counts five times its rows, and the dictionary is the one list."""
    db = store.DB(None, "delta_strings")
    table = f"delta_shared_{name}"
    _fresh(store, db, table)
    try:
        encs = ["dba"] if name in ds.FRONT_BY_NAME else ["dlba", "dba"]
        for enc in encs:
            store.engine.put_parquet(table, ds.file_of(name, enc))
        store.engine.put_parquet(table, ds.plain_of(name))
        store.engine.put_parquet(table, ds.twin_of(name))
        store.engine.put_arrow(table, ds.record_of(name))
        k = len(encs) + 3
        got = groups(run(db, table, lambda q: q.Aggregate([lp.Count(V), lp.Sum(V)], [S])), ["s"], [lp.Count(V), lp.Sum(V)])
        exp = {key: (k * v[1], k * v[0]) for key, v in reference(name, lambda c, i: True, ["s"]).items()}
        same(got, exp, name)
        assert store.engine.dict_export(table, "s") == [v.encode() for v in ds.first_occurrence(ds.table(name).column("s").to_pylist())]
    finally:
        store.engine.drop_table(table)
        db.tables.pop(table, None)


@pytest.mark.parametrize("name,enc", ds.CASES, ids=ds.CASE_IDS)
def test_group_by_and_leaves_match_the_twin_and_pyarrow(store, parts, name, enc):
    db, made = parts
    plans = [(None, lambda c, i: True)] + filters(name)
    for filt, pred in plans:
        build = (lambda q: q.Filter(filt).Aggregate(AGGS, [S])) if filt is not None else (lambda q: q.Aggregate(AGGS, [S]))
        exp = reference(name, pred, ["s"])
        what = f"{name}-{enc} {filt.Name() if filt is not None else None}"
        for kind in ("twin", "eager", "borrow"):
            same(groups(run(db, made[(name, enc, kind)], build), ["s"], AGGS), exp, f"{what} {kind}")
        build2 = (lambda q: q.Filter(filt).Aggregate([lp.Count(V)], [])) if filt is not None else (lambda q: q.Aggregate([lp.Count(V)], []))
        n = sum(v[1] for v in exp.values())
        got = groups(run(db, made[(name, enc, "eager")], build2), [], [lp.Count(V)])
        assert got.get((), (0,))[0] == n, what


@pytest.mark.parametrize("name,enc", [("v2_optional", "dlba"), ("collisions", "dba"), ("many_small_pages", "dba"),
                                      ("sorted_prefixes", "dba"), ("page_edges", "dba")])
def test_kernel_routing_equals_the_twins(store, parts, name, enc):
    _, made = parts
    lit = literal(name)
    aggs = [lp.Sum(V), lp.Count(V), lp.Min(V), lp.Max(V)]
    route = ("row_groups", "row_groups_tiles", "row_groups_runs")
    for filt in (None, S.Eq(lp.Literal(lit)), lp.Or(S.Eq(lp.Literal(lit)), V.Lt(lp.Literal(-900)))):
        st = stats_of(store, made[(name, enc, "eager")], filt, ["s"], aggs)
        # (the dictionary twin of a sorted layout holds runs that the sorted-run kernel may take)
        for kind in ("plain",) if name in ds.FRONT_BY_NAME else ("twin", "plain"):
            tw = stats_of(store, made[(name, enc, kind)], filt, ["s"], aggs)
            assert [st[k] for k in route] == [tw[k] for k in route], (kind, st, tw)


@pytest.mark.parametrize("name,enc", ds.CASES, ids=ds.CASE_IDS)
def test_distinct_and_hash_keys(parts, name, enc):
    db, made = parts
    exp = {(v,) for v in ds.table(name).column("s").to_pylist() if v is not None}
    seen = {}
    for kind in ("eager", "borrow", "twin"):
        got = []
        for b in run(db, made[(name, enc, kind)], lambda q: q.Distinct(S)):
            got.extend((v,) for v in as_strings(b.column(b.schema.get_field_index("s"))))
        assert len(got) == len(set(got)), kind
        seen[kind] = set(got)
        assert seen[kind] - {(None,)} == exp, kind
    assert seen["eager"] == seen["borrow"] == seen["twin"]
    exp2 = reference(name, lambda c, i: True, ["s", "value"])
    got2 = groups(run(db, made[(name, enc, "eager")], lambda q: q.Aggregate([lp.Count(V)], [S, V])), ["s", "value"], [lp.Count(V)])
    same(got2, {k: (v[1],) for k, v in exp2.items()}, f"{name}-{enc} (s, value)")


@pytest.mark.parametrize("name,enc", ds.CASES, ids=ds.CASE_IDS)
def test_filter_only_plans(store, parts, name, enc):
    db, made = parts
    t = ds.table(name)
    cols = {n: t.column(n).to_pylist() for n in t.column_names}
    for filt, pred in filters(name):
        sel = [i for i in range(t.num_rows) if pred(cols, i)]
        for kind in ("eager", "borrow"):
            table = made[(name, enc, kind)]
            assert rows_of(db, table, filt, ["timestamp", "s"]) == [(cols["timestamp"][i], cols["s"][i]) for i in sel], (kind, filt.Name())
            assert rows_of(db, table, filt, ["timestamp", "value"]) == [(cols["timestamp"][i], cols["value"][i]) for i in sel], (kind, filt.Name())
        if filt.Op == lp.OpOr:
            continue
        assert launches(store, made[(name, enc, "eager")], filt, ["timestamp", "value"]) == \
            launches(store, made[(name, enc, "twin")], filt, ["timestamp", "value"]), filt.Name()


@pytest.mark.parametrize("borrow", [False, True])
def test_dictionary_pages_followed_by_delta_and_plain_pages(store, borrow):
    import numpy as np
    db = store.DB(None, "delta_strings")
    table = f"delta_mixed_{int(borrow)}"
    db.Table(table, two_columns())
    buf = ds.mixed_file()
    arr = np.frombuffer(buf, dtype=np.uint8)
    try:
        store.engine.put_parquet(table, arr, borrow=borrow)
        s = ds.mixed_strings()
        assert as_strings(store.engine.decode_column(table, 0, "s")) == s
        dict_vals = [f"dict/{i:03d}" for i in range(20)]
        exp = dict_vals + [v for v in ds.first_occurrence(s) if v not in dict_vals]
        assert store.engine.dict_export(table, "s") == [v.encode() for v in exp]
        got = groups(run(db, table, lambda q: q.Aggregate([lp.Count(lp.Col("timestamp"))], [S])), ["s"], [lp.Count(lp.Col("timestamp"))])
        assert got == {(v,): (s.count(v),) for v in set(s)}
    finally:
        store.engine.drop_table(table)
        db.tables.pop(table, None)


@pytest.mark.parametrize("case", ["dlba_sum", "long_prefix", "bit_width"])
def test_corrupted_chunk_fails_only_the_queries_that_touch_it(store, case):
    import numpy as np
    name, buf, message = next(c for c in ds.corrupted() if c[0] == case)
    db = store.DB(None, "delta_strings")
    for borrow in (False, True):
        table = f"delta_corrupt_{case}_{int(borrow)}"
        db.Table(table, two_columns())
        try:
            store.engine.put_parquet(table, np.frombuffer(buf, dtype=np.uint8), borrow=borrow)
            ts = lp.Col("timestamp")
            got = groups(run(db, table, lambda q: q.Aggregate([lp.Count(ts), lp.Sum(ts)], [])), [], [lp.Count(ts), lp.Sum(ts)])
            assert got == {(): (152, sum(range(152)))}
            with pytest.raises(_lib.FrostGPUError, match=re.escape("column s: " + message)):
                run(db, table, lambda q: q.Aggregate([lp.Count(ts)], [S]))
            with pytest.raises(_lib.FrostGPUError, match=re.escape(message)):
                run(db, table, lambda q: q.Filter(S.Eq(lp.Literal("ok-1"))).Aggregate([lp.Count(ts)], []))
        finally:
            store.engine.drop_table(table)
            db.tables.pop(table, None)


def test_front_coded_values_get_their_own_ids(store, parts):
    """The chain: 1 200 values each extending the previous one, then one with prefix 0; every value its own id."""
    _, made = parts
    s = ds.table("long_chain").column("s").to_pylist()
    got = store.engine.decode_column(made[("long_chain", "dba", "eager")], 0, "s")
    assert as_strings(got) == s
    if pa.types.is_dictionary(got.type):
        by_value = {}
        for v, i in zip(s, got.indices.to_pylist()):
            assert by_value.setdefault(v, i) == i, v
        assert len(set(by_value.values())) == len(by_value) == 1201
