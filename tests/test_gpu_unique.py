"""Unique(int64) on the GPU path: the reference's golden through query.NewEngine, seeded parts against the plain
reference (tests/unique_reference.py) in every int64 encoding the engine reads, dense and hash tables, routing to the
general scan kernel, caching, the multi-rank merge, the Arrow export and the refusals."""
import ctypes as C
import io

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

from frostdb_b200 import _lib, query
from frostdb_b200 import dynparquet as dp
from frostdb_b200 import logicalplan as lp
from frostdb_b200.physicalplan import GPUScan
from frostdb_b200.store import GPUEngine
from tests import unique_reference as ref
from tests.bool_keys_reference import read_part
from tests.golden import unique_aggregation as golden
from tests.util import label_values, rows_of

pytestmark = pytest.mark.gpu

L = lp.Literal
A, B, K, T, V, U, W = (lp.Col(c) for c in ("labels.a", "labels.b", "k", "timestamp", "value", "u", "w"))
I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
N_PART, RG, PARTS_T0 = 6000, 2000, (0, 10_000, 20_000)
ENCODINGS = ["plain_required", "plain_optional", "dict64", "delta", "lz4"]
FLIP = 1000  # `value` of the rows whose `u` differs from the rest of their group (every other `value` is below it)


def _bucket():
    return lp.Mul(lp.Div(T, L(1000)), L(1000)).Alias("bucket")


def _key_fn(k):
    if isinstance(k, lp.AliasExpr):  # (timestamp / 1000) * 1000, timestamps are not negative
        return lambda part, i: (part["timestamp"][i] // 1000) * 1000
    return lambda part, i: part[k.ColumnName][i]


def _columns(p, enc, edges):
    """Part p: `u` and `w` are constant per labels.a value in a part; labels.a == 1 differs across parts; a few rows
    (value == FLIP) differ inside their group; with NULLs, labels.a == 3 has some NULL `u` rows and `w` is NULL
    everywhere but one row."""
    rng = np.random.default_rng(500 + p)
    n = N_PART
    pool = np.array([I64_MIN, I64_MIN + 1, I64_MAX - 1, I64_MAX] if edges else [-5, 7, 11, 40, 1 << 40], dtype=np.int64)
    a = rng.integers(0, 5, n).astype(np.int32)
    a[rng.random(n) < 0.1] = -1
    base = pool[[0, 1, 2, 3, 1]].copy()
    base[1] = pool[p % len(pool)]  # labels.a == 1: equal inside each part, different across parts
    u = np.where(a < 0, pool[3], base[np.maximum(a, 0)])
    value = rng.integers(0, 1000, n).astype(np.int64)
    flip = np.flatnonzero(a == 2)[:1] if p == 1 else np.flatnonzero(a == 4)[:2]
    u[flip] = pool[0] if u[flip[0]] != pool[0] else pool[1]
    value[flip] = FLIP
    nulls = np.zeros(n, bool)
    if enc != "plain_required":
        nulls[np.flatnonzero(a == 3)[::50]] = True
    w = np.full(n, pool[2], np.int64)
    cols = {
        "labels.a": (a, label_values(5)), "labels.b": (rng.integers(0, 3, n).astype(np.int32), label_values(3)),
        "timestamp": PARTS_T0[p] + np.arange(n, dtype=np.int64), "value": value,
        "k": rng.integers(0, 40, n).astype(np.int64) * 1_000_003,
        "u": pa.array(u, mask=nulls if nulls.any() else None),
        "w": pa.array(w, mask=(np.arange(n) != 17) if enc != "plain_required" else None),
    }
    return cols


def _write(cols, enc):
    """One part, `u` and `w` in encoding `enc`: REQUIRED or OPTIONAL PLAIN, an int64 dictionary chunk,
    DELTA_BINARY_PACKED, or PLAIN under LZ4_RAW (every column)."""
    fields, arrays = [], []
    for name in sorted(cols):
        v = cols[name]
        if isinstance(v, tuple):
            idx, d = v
            arr = pa.DictionaryArray.from_arrays(pa.array(np.maximum(idx, 0), mask=idx < 0), pa.array(d))
        else:
            arr = v if isinstance(v, pa.Array) else pa.array(v)
        nullable = name.startswith("labels.") or (name in ("u", "w") and enc != "plain_required")
        fields.append(pa.field(name, arr.type, nullable=nullable))
        arrays.append(arr)
    t = pa.Table.from_arrays(arrays, schema=pa.schema(fields)).replace_schema_metadata({"dynamic_columns": "labels:a,b"})
    dict_cols = ["labels.a", "labels.b"] + (["u", "w"] if enc == "dict64" else [])
    plain = {c: "PLAIN" for c in cols if c not in dict_cols}
    if enc == "delta":
        plain["u"] = plain["w"] = "DELTA_BINARY_PACKED"
    sink = io.BytesIO()
    pq.write_table(t, sink, compression="LZ4" if enc == "lz4" else "NONE", use_dictionary=dict_cols, column_encoding=plain,
                   data_page_version="2.0", row_group_size=RG, store_schema=False)
    return sink.getvalue()


_ENGINES = {}


def _seeded(enc, edges):
    key = (enc, edges)
    if key not in _ENGINES:
        bufs = [_write(_columns(p, enc, edges), enc) for p in range(len(PARTS_T0))]
        e = GPUEngine(0)
        for b in bufs:
            e.put_parquet("u", b)
        _ENGINES[key] = (e, [read_part(b) for b in bufs], bufs)
    return _ENGINES[key]


@pytest.fixture(scope="module", autouse=True)
def _close_engines(built_lib):
    yield
    for e, _, _ in _ENGINES.values():
        e.close()
    _ENGINES.clear()


def _run(e, keys, aggs, filt=None, table="u"):
    """Executes one aggregate plan; returns (records, stats)."""
    lib = _lib.load()
    scan = GPUScan(e, table, filt, _lib.PLAN_AGGREGATE, keys, list(aggs))
    q, keep = scan.prepare()
    try:
        res = C.c_void_p()
        _lib.check(lib.fgpu_query_execute(e.handle, q, e.table_watermark(table), C.byref(res)))
        try:
            return [scan.renamed(b) for b in e.drain(res)], e.stats(res)
        finally:
            lib.fgpu_result_free(res)
    finally:
        lib.fgpu_query_free(q)
        del keep


def _names(keys, aggs):
    return [k.AliasName if isinstance(k, lp.AliasExpr) else k.Name() for k in keys] + [a.Name() for a in aggs]


def _selected(filt):
    if filt is None:
        return None
    from tests.bool_keys_reference import eval_bool
    return lambda part, i: eval_bool(filt, part, i)


def _expected(parts, keys, cols, filt=None):
    return ref.rows(parts, [_key_fn(k) for k in keys], cols, _selected(filt))


def _rows_at(got, idx):
    """Result rows of the columns at positions idx (a plan may name two columns alike), sorted as rows_of sorts."""
    out = []
    for b in got:
        cols = [b.column(i).dictionary_decode() if pa.types.is_dictionary(b.column(i).type) else b.column(i) for i in idx]
        out.extend(zip(*[[v.decode() if isinstance(v, bytes) else v for v in c.to_pylist()] for c in cols]))
    return sorted(out, key=lambda r: tuple((x is None, x) for x in r))


def _check_general_scan(st):
    assert st["row_groups_runs"] == st["row_groups_prefix"] == st["row_groups_tiles"] == 0
    assert st["row_groups"] > 0


def _check(got, parts, keys, cols, filt=None):
    aggs = [lp.Unique(lp.Col(c)) for c in cols]
    for b in got:
        for a in aggs:
            arr = b.column(b.schema.get_field_index(a.Name()))
            assert arr.type == pa.int64()
            assert arr.null_count == sum(x is None for x in arr.to_pylist())
            if arr.null_count == 0:
                assert arr.buffers()[0] is None
    assert rows_of(got, _names(keys, aggs)) == _expected(parts, keys, cols, filt)


# ---- the reference's golden ------------------------------------------------------------------------------------
@pytest.mark.parametrize("how", ["parquet", "arrow"])
def test_golden(store, how):
    db = store.DB(None, "golden_unique")
    name = "gu_" + how
    if name in db.tables:
        store.engine.drop_table(name)
        db.tables.pop(name)
    schema = dp.Schema("test", [dp.ColumnDefinition(c, dp.TYPE_INT64) for c, _ in golden.SCHEMA], [])
    t = db.Table(name, schema)
    if how == "parquet":
        t.Insert({c: np.array(v, np.int64) for c, v in golden.ROWS.items()}, sort=False)
    else:
        t.InsertRecord(pa.RecordBatch.from_arrays([pa.array(golden.ROWS[c], pa.int64()) for c, _ in golden.SCHEMA],
                                                  names=[c for c, _ in golden.SCHEMA]))
    out = []
    func, col = golden.AGGREGATE
    assert func == "unique"
    query.NewEngine(None, db.TableProvider()).ScanTable(name).Aggregate([lp.Unique(lp.Col(col))], [lp.Col(c) for c in golden.GROUP_BY]) \
        .Execute(None, lambda ctx, r: out.append(r))
    names = list(golden.EXPECTED)
    assert rows_of(out, names) == sorted(zip(*golden.EXPECTED.values()), key=lambda r: tuple((x is None, x) for x in r))
    col_u = out[0].column(out[0].schema.get_field_index("unique(example)"))
    assert col_u.type == pa.int64() and col_u.null_count == 1


# ---- seeded parts ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("edges", [False, True], ids=["small", "int64_ends"])
@pytest.mark.parametrize("enc", ENCODINGS)
def test_dense_tables(enc, edges):
    e, parts, _ = _seeded(enc, edges)
    for keys in ([A], [A, B], [B]):
        got, st = _run(e, keys, [lp.Unique(U), lp.Unique(W)])
        _check(got, parts, keys, ["u", "w"])
        _check_general_scan(st)


@pytest.mark.parametrize("edges", [False, True], ids=["small", "int64_ends"])
@pytest.mark.parametrize("enc", ENCODINGS)
def test_hash_tables(enc, edges):
    e, parts, _ = _seeded(enc, edges)
    for keys in ([K], [A, K], [_bucket()], [A, _bucket()]):
        got, st = _run(e, keys, [lp.Unique(U)])
        _check(got, parts, keys, ["u"])
        _check_general_scan(st)


@pytest.mark.parametrize("enc", ["plain_optional", "dict64"])
def test_filters_and_pruned_row_groups(enc):
    e, parts, _ = _seeded(enc, False)
    drop_flips = V.Lt(L(FLIP))
    got, _ = _run(e, [A], [lp.Unique(U)])
    assert any(r[1] is None for r in rows_of(got))
    for filt in (drop_flips, T.GtEq(L(PARTS_T0[1])), lp.And(T.GtEq(L(PARTS_T0[1] + 2500)), drop_flips),
                 A.Eq(L("v000002")), T.Lt(L(PARTS_T0[1] + 10))):
        got, st = _run(e, [A, B], [lp.Unique(U)], filt)
        _check(got, parts, [A, B], ["u"], filt)
        _check_general_scan(st)
        if filt.Name().startswith("timestamp"):
            assert st["row_groups_pruned"] > 0
    # removing the only differing rows makes labels.a == 2 and 4 groups (no NULLs there) take their value
    got, _ = _run(e, [A], [lp.Unique(U)], drop_flips)
    by_a = dict((r[0], r[1]) for r in rows_of(got))
    assert by_a["v000002"] is not None and by_a["v000004"] is not None


def test_with_the_other_aggregates():
    e, parts, _ = _seeded("plain_optional", True)
    others = [lp.Sum(V), lp.Count(V), lp.Min(V), lp.Max(T)]
    for keys in ([A, B], [K]):
        plain, _ = _run(e, keys, others)
        # 8 stored cells and Counts: the budget exactly
        mixed, st = _run(e, keys, [lp.Sum(V), lp.Unique(U), lp.Count(V), lp.Min(V), lp.Unique(W), lp.Max(T)])
        _check_general_scan(st)
        nk = len(keys)
        keep = list(range(nk))
        assert _rows_at(mixed, keep + [nk + i for i in (0, 2, 3, 5)]) == _rows_at(plain, keep + [nk + i for i in range(4)])
        assert _rows_at(mixed, keep + [nk + 1, nk + 4]) == _expected(parts, keys, ["u", "w"])
        assert [f.type for f in mixed[0].schema][nk:] == [pa.int64()] * 6
        same, _ = _run(e, keys, [lp.Unique(U), lp.Count(V), lp.Unique(U)])  # two Uniques of one column
        assert _rows_at(same, keep + [nk]) == _rows_at(same, keep + [nk + 2]) == _expected(parts, keys, ["u"])
    assert _refusal(e, [A], [lp.Unique(U)] * 4 + [lp.Count(V)]) == (_lib.FGPU_ERR_UNSUPPORTED, "too many aggregates")
    _run(e, [A], [lp.Unique(U)] * 3 + [lp.Sum(V), lp.Count(V)])  # 8 stored cells and Counts: accepted


def test_avg_next_to_unique_through_the_builder(store):
    db = store.DB(None, "unique_avg")
    name = "ua"
    if name not in db.tables:
        schema = dp.SampleDefinition()
        schema.columns.append(dp.ColumnDefinition("u", dp.TYPE_INT64, nullable=True))
        t = db.Table(name, schema)
        rng = np.random.default_rng(9)
        n = 5000
        a = rng.integers(0, 4, n).astype(np.int32)
        u = np.where(a == 0, 7, np.where(a == 1, I64_MIN, rng.integers(0, 3, n))).astype(np.int64)
        t.Insert({"example_type": (np.zeros(n, np.int32), ["cpu"]), "stacktrace": (np.zeros(n, np.int32), ["s"]),
                  "labels.a": (a, label_values(4)), "timestamp": np.arange(n, dtype=np.int64),
                  "value": rng.integers(-50, 50, n).astype(np.int64),
                  "u": [None if m else int(x) for x, m in zip(u, (a == 3) & (np.arange(n) % 97 == 0))]},
                 row_group_size=1024)
    out = []
    query.NewEngine(None, db.TableProvider()).ScanTable(name).Aggregate([lp.Avg(V), lp.Unique(U)], [A]).Limit(L(10)) \
        .Execute(None, lambda ctx, r: out.append(r))
    rows = {r[0]: r[1:] for r in rows_of(out, ["labels.a", "avg(value)", "unique(u)"])}
    assert rows["v000000"][1] == 7 and rows["v000001"][1] == I64_MIN
    assert rows["v000002"][1] is None and rows["v000003"][1] is None
    assert all(isinstance(v[0], int) for v in rows.values())


# ---- routing ---------------------------------------------------------------------------------------------------
def _sorted_engine():
    schema = dp.SampleDefinition()
    schema.columns.append(dp.ColumnDefinition("u", dp.TYPE_INT64))
    e = GPUEngine(0)
    parts = []
    for p in range(2):
        rng = np.random.default_rng(40 + p)
        n = 60_000
        a = rng.integers(0, 4, n).astype(np.int32)
        cols = {"example_type": (np.zeros(n, np.int32), ["cpu"]), "stacktrace": (rng.integers(0, 3, n).astype(np.int32), label_values(3)),
                "labels.a": (a, label_values(4)), "labels.b": (rng.integers(0, 3, n).astype(np.int32), label_values(3)),
                "timestamp": p * n + np.arange(n, dtype=np.int64), "value": rng.integers(0, 1000, n).astype(np.int64),
                "u": np.where(a == 1, 5 + p, 9).astype(np.int64)}
        b = dp.write_part(schema, cols, row_group_size=20_000)
        e.put_parquet("s", b)
        parts.append(read_part(b))
    return e, parts


def test_routing_on_sorted_parts(monkeypatch):
    e, parts = _sorted_engine()
    try:
        base = [lp.Sum(V), lp.Count(V)]
        for filt in (None, T.GtEq(L(30_000))):
            got, st = _run(e, [A, B], base, filt, table="s")
            assert st["row_groups_runs"] + st["row_groups_tiles"] > 0
            got_u, st_u = _run(e, [A, B], base + [lp.Unique(U)], filt, table="s")
            _check_general_scan(st_u)
            names = _names([A, B], base)
            assert rows_of(got_u, names) == rows_of(got, names)
            assert rows_of(got_u, _names([A, B], [lp.Unique(U)])) == _expected(parts, [A, B], ["u"], filt)
    finally:
        e.close()


# ---- caching -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("switch", [None, "FROSTGPU_NO_EXEC_CACHE", "FROSTGPU_NO_PLAN_CACHE"])
def test_prepared_plan_executes_alike(switch, monkeypatch):
    if switch:
        monkeypatch.setenv(switch, "1")
    e, parts, _ = _seeded("plain_optional", True)
    lib = _lib.load()
    for keys in ([A, B], [K]):
        aggs = [lp.Unique(U), lp.Count(V), lp.Unique(W)]
        q, keep = GPUScan(e, "u", None, _lib.PLAN_AGGREGATE, keys, aggs).prepare()
        try:
            seen = []
            for _ in range(3):  # compiled, then the cached Execute (dense tables)
                res = C.c_void_p()
                _lib.check(lib.fgpu_query_execute(e.handle, q, e.table_watermark("u"), C.byref(res)))
                try:
                    got = list(e.drain(res))
                finally:
                    lib.fgpu_result_free(res)
                _check(got, parts, keys, ["u", "w"])
                seen.append(rows_of(got))
            assert seen[0] == seen[1] == seen[2]
        finally:
            lib.fgpu_query_free(q)
            del keep


# ---- multi-rank --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_ranks", [2, 3])
@pytest.mark.parametrize("mode", ["dense", "hash"])
def test_multirank_collective(n_ranks, mode):
    """Ranks are contexts on one GPU, one part each (the parts of the seeded set): labels.a == 1 is constant on each
    rank and different across them (NULL), labels.a == 0 is constant everywhere (its value), and labels.a == 3 has
    NULL rows on the ranks that hold them."""
    from frostdb_b200.store import comm_setup
    _, parts, bufs = _seeded("plain_optional", False)
    bufs, parts = bufs[:n_ranks], parts[:n_ranks]
    keys = [A, B] if mode == "dense" else [A, K]
    aggs = [lp.Unique(U), lp.Count(V), lp.Unique(W)]
    exp = _expected(parts, keys, ["u", "w"])
    names = _names(keys, aggs)
    lib = _lib.load()
    engines = [GPUEngine(0) for _ in range(n_ranks)]
    prepared, pend, opened = [], [], False
    try:
        for e, b in zip(engines, bufs):
            for col, card in (("labels.a", 5), ("labels.b", 3)):
                e.dict_preload("mr", col, [v.encode() for v in label_values(card)])
            e.put_parquet("mr", b)
        comm_setup(engines, slot_bytes=16 << 20)
        opened = True
        prepared = [GPUScan(e, "mr", None, _lib.PLAN_AGGREGATE, keys, aggs).prepare() for e in engines]
        for rep in range(2):  # compiled plan, then the cached one
            pend = [e.execute_collective_begin(p[0], e.table_watermark("mr")) for e, p in zip(engines, prepared)]
            for r, e in enumerate(engines):
                e.execute_collective_end(pend[r])
                got = list(e.drain(pend[r]))
                assert rows_of(got, names[:len(keys)] + names[len(keys)::2]) == exp, (r, rep)
            for res in pend:
                lib.fgpu_result_free(res)
            pend = []
        by_a = {}
        for row in exp:
            by_a.setdefault(row[0], set()).add(row[len(keys)])
        assert by_a["v000001"] == {None} and None not in by_a["v000000"]
    finally:
        for res in pend:
            lib.fgpu_result_free(res)
        for q, _ in prepared:
            lib.fgpu_query_free(q)
        for e in engines:
            if opened:
                e.comm_close()
            e.close()


# ---- refusals ----------------------------------------------------------------------------------------------------
def _refusal(e, keys, aggs, table="u"):
    with pytest.raises(_lib.FrostGPUError) as ei:
        _run(e, keys, aggs, table=table)
    return ei.value.code, ei.value.msg


def test_refusals(store):
    e, _, _ = _seeded("plain_required", False)
    assert _refusal(e, [A], [lp.Unique(lp.Add(V, L(1)))])[0] == _lib.FGPU_ERR_UNSUPPORTED
    assert _refusal(e, [A], [lp.Unique(A)])[0] == _lib.FGPU_ERR_UNSUPPORTED
    db = store.DB(None, "unique_refusals")
    if "ur" not in db.tables:
        t = db.Table("ur", dp.SampleDefinitionWithFloat())
        n = 100
        base = {"example_type": (np.zeros(n, np.int32), ["cpu"]), "stacktrace": (np.zeros(n, np.int32), ["s"]),
                "labels.a": (np.zeros(n, np.int32), ["x"]), "timestamp": np.arange(n, dtype=np.int64),
                "value": np.ones(n, np.int64)}
        t.Insert(dict(base, floatvalue=np.ones(n)))
        t.Insert(base)  # a part without floatvalue
    eng = store.engine
    code, _ = _refusal(eng, [A], [lp.Unique(lp.Col("floatvalue"))], table="ur")
    assert code == _lib.FGPU_ERR_UNSUPPORTED
    assert _refusal(eng, [A], [lp.Sum(lp.Col("nosuch"))], table="ur")[0] == _refusal(eng, [A], [lp.Unique(lp.Col("nosuch"))], table="ur")[0] \
        == _lib.FGPU_ERR_NOT_FOUND
    db2 = store.DB(None, "unique_missing")
    if "um" not in db2.tables:
        s = dp.SampleDefinition()
        s.columns.append(dp.ColumnDefinition("u", dp.TYPE_INT64))
        t2 = db2.Table("um", s)
        n = 100
        base = {"example_type": (np.zeros(n, np.int32), ["cpu"]), "stacktrace": (np.zeros(n, np.int32), ["s"]),
                "labels.a": (np.zeros(n, np.int32), ["x"]), "timestamp": np.arange(n, dtype=np.int64), "value": np.ones(n, np.int64)}
        t2.Insert(dict(base, u=np.full(n, 4, np.int64)))
        t2.Insert(base)  # `u` missing from this part's row groups
    assert _refusal(eng, [A], [lp.Unique(U)], table="um")[0] == _lib.FGPU_ERR_NOT_FOUND
