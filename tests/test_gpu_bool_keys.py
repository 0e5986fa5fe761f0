"""Distinct over boolean expression keys (`Distinct(labels.a, value > 0)`) on the GPU path: the reference's goldens,
seeded parts against the plain reference (tests/bool_keys_reference.py), routing, caching, the multi-rank merge and
the refusals a boolean key shares with the filter."""
import ctypes as C

import numpy as np
import pyarrow as pa
import pytest

from frostdb_b200 import _lib, query
from frostdb_b200 import dynparquet as dp
from frostdb_b200 import logicalplan as lp
from frostdb_b200.physicalplan import GPUScan
from frostdb_b200.store import GPUEngine
from tests import bool_keys_reference as ref
from tests import golden_runner as gr
from tests.golden.logictest_distinct_proj import CASES
from tests.util import label_values, rows_of

pytestmark = pytest.mark.gpu

L = lp.Literal
V, F, T = lp.Col("value"), lp.Col("floatvalue"), lp.Col("timestamp")
A, B, CC, NOSUCH = lp.Col("labels.a"), lp.Col("labels.b"), lp.Col("labels.c"), lp.Col("labels.nosuch")
N = lp.Col("nullint")  # a nullable int64 column (values 1 .. 1000, so that no NULL key meets a real 0)
N_PART, PARTS_T0 = 6000, (0, 10_000, 20_000)

# one leaf kind each (numeric, float, dictionary, nesting, absent columns under every operator class)
KEYS = {
    "int_gt": V.Gt(L(500)), "int_ge": V.GtEq(L(999)), "int_lt": V.Lt(L(0)), "int_le": V.LtEq(L(3)),
    "int_eq": V.Eq(L(7)), "int_ne": V.NotEq(L(7)), "ts_gt": T.Gt(L(12_000)), "ts_lt": T.Lt(L(15_000)),
    "nint_gt": N.Gt(L(500)), "nint_ne": N.NotEq(L(5)), "nint_eq_null": N.Eq(L(None)),
    "float_gt": F.Gt(L(500.5)), "float_ne_nan": F.NotEq(L(float("nan"))), "float_eq_nan": F.Eq(L(float("nan"))),
    "dict_eq": A.Eq(L("v000001")), "dict_ne": A.NotEq(L("v000001")), "dict_eq_null": A.Eq(L(None)),
    "dict_ne_null": A.NotEq(L(None)), "dict_contains": A.Contains("2"), "dict_not_contains": A.ContainsNot("2"),
    "dict_regex": A.RegexMatch("0[34]$"), "partial_label": CC.Eq(L("v000001")),
    "and": lp.And(V.Gt(L(300)), A.Eq(L("v000000"))), "or": lp.Or(T.Lt(L(3000)), B.NotEq(L(None))),
    "nested": lp.Or(lp.And(V.Lt(L(100)), B.Eq(L("v000002"))), lp.And(F.GtEq(L(900.0)), CC.NotEq(L(None)))),
    "nosuch_gt": NOSUCH.Gt(L(0)), "nosuch_eq_int": NOSUCH.Eq(L(5)), "nosuch_eq_str": NOSUCH.Eq(L("x")),
    "nosuch_ne_null": NOSUCH.NotEq(L(None)), "nosuch_regex": NOSUCH.RegexMatch("^$"), "nosuch_contains": NOSUCH.Contains("x"),
}


def _parts():
    schema = dp.SampleDefinitionWithFloat()
    schema.columns.append(dp.ColumnDefinition("nullint", dp.TYPE_INT64, nullable=True))
    bufs = []
    for p, t0 in enumerate(PARTS_T0):
        rng = np.random.default_rng(100 + p)
        n = N_PART
        f = rng.integers(0, 10**6, n).astype(np.float64) / 1000.0
        cols = {
            "example_type": (np.zeros(n, np.int32), ["cpu"]),
            "stacktrace": (rng.integers(0, 3, n).astype(np.int32), ["s0", "s1", "s2"]),
            "timestamp": t0 + np.arange(n, dtype=np.int64),
            "value": rng.integers(0, 1000, n).astype(np.int64),
            "floatvalue": pa.array(f, mask=rng.random(n) < 0.1),
            "nullint": pa.array(rng.integers(1, 1001, n).astype(np.int64), mask=rng.random(n) < 0.15),
        }
        for name, card, pnull in (("a", 6, 0.1), ("b", 3, 0.2)) + ((("c", 4, 0.3),) if p != 1 else ()):
            idx = rng.integers(0, card, n).astype(np.int32)
            idx[rng.random(n) < pnull] = -1
            cols[f"labels.{name}"] = (idx, label_values(card))
        bufs.append(dp.write_part(schema, cols, row_group_size=1500))
    return schema, bufs


@pytest.fixture(scope="module")
def seeded(built_lib):
    _, bufs = _parts()
    e = GPUEngine(0)
    for b in bufs:
        e.put_parquet("bk", b)
    yield e, [ref.read_part(b) for b in bufs], bufs
    e.close()


def _run(e, table, keys, filt=None, kind=_lib.PLAN_DISTINCT, aggs=()):
    """Executes one plan; returns (records, stats)."""
    lib = _lib.load()
    scan = GPUScan(e, table, filt, kind, keys, list(aggs))
    q, keep = scan.prepare()
    try:
        res = C.c_void_p()
        _lib.check(lib.fgpu_query_execute(e.handle, q, e.table_watermark(table), C.byref(res)))
        try:
            return list(e.drain(res)), e.stats(res)
        finally:
            lib.fgpu_result_free(res)
    finally:
        lib.fgpu_query_free(q)
        del keep


def _expected(parts, keys, filt=None):
    """The reference's rows, with a NULL int64 key as the engine returns it: 0, the value NULL hashes alike with
    (dynparquet/hashed.go:254-262)."""
    rows = ref.distinct_rows(parts, keys, filt)
    ints = [i for i, k in enumerate(keys) if isinstance(k, lp.Column) and k.ColumnName in ("value", "nullint")]
    rows = {tuple(0 if (i in ints and x is None) else x for i, x in enumerate(r)) for r in rows}
    return sorted(rows, key=lambda r: tuple((x is None, x) for x in r))


def _check(got, parts, keys, filt=None):
    names = [k.Name() for k in keys]
    for b in got:
        assert b.schema.names == names
        for k, a in zip(keys, b.columns):
            if isinstance(k, lp.BinaryExpr):
                assert a.type == pa.bool_() and a.null_count == 0
    assert rows_of(got, names) == _expected(parts, keys, filt)


@pytest.mark.parametrize("no_prune", [False, True])
@pytest.mark.parametrize("case", CASES, ids=[c["source"].split("/")[-1] for c in CASES])
def test_goldens(store, case, no_prune, monkeypatch):
    if no_prune:
        monkeypatch.setenv("FROSTGPU_NO_PRUNE", "1")
    db = store.DB(None, "golden_bool")
    name = "gb_" + case["source"].split("/")[-1] + ("_np" if no_prune else "")
    if name in db.tables:
        store.engine.drop_table(name)
        db.tables.pop(name)
    ran = 0
    for ex, got, exp in gr.run_case(case, lambda schema: db.Table(name, schema),
                                    lambda: query.NewEngine(None, db.TableProvider()).ScanTable(name)):
        gr.check(ex, got, exp)
        ran += 1
    assert ran > 0


@pytest.mark.parametrize("key", list(KEYS), ids=list(KEYS))
def test_key_alone_and_with_dictionary_keys(seeded, key):
    e, parts, _ = seeded
    k = KEYS[key]
    for keys in ([k], [A, B, k]):
        got, st = _run(e, "bk", keys)
        _check(got, parts, keys)
        assert st["row_groups_runs"] == 0 and st["row_groups_tiles"] == 0


@pytest.mark.parametrize("key", ["int_gt", "ts_gt", "dict_eq_null", "nested", "nosuch_eq_int", "partial_label", "nint_gt",
                                 "nint_eq_null"])
def test_key_with_int64_key(seeded, key):
    e, parts, _ = seeded
    for keys in ([V, KEYS[key]], [N, KEYS[key]], [A, N, KEYS[key]]):  # hash tables; N has NULL keys
        got, st = _run(e, "bk", keys)
        _check(got, parts, keys)
        assert st["row_groups_runs"] == 0 and st["row_groups_tiles"] == 0


def test_two_boolean_keys_filters_and_no_prune(seeded, monkeypatch):
    e, parts, _ = seeded
    plans = [([A, KEYS["int_gt"], KEYS["dict_regex"]], None),
             ([A, KEYS["ts_gt"]], T.GtEq(L(10_000))),         # the filter drops every row group of the first part
             ([A, KEYS["ts_gt"]], lp.And(T.GtEq(L(10_000)), V.Lt(L(900)))),
             ([A, KEYS["and"]], KEYS["and"]),                 # the same expression as filter and key: always true
             ([B, KEYS["ts_lt"], V], A.NotEq(L(None)))]
    for keys, filt in plans:
        got, st = _run(e, "bk", keys, filt)
        _check(got, parts, keys, filt)
        if filt is not None and filt.Name() == keys[1].Name():
            assert all(r[1] is True for r in rows_of(got))
    monkeypatch.setenv("FROSTGPU_NO_PRUNE", "1")
    for keys, filt in plans:
        got, st = _run(e, "bk", keys, filt)
        assert st["row_groups_pruned"] == 0
        _check(got, parts, keys, filt)


def test_statistics_decide_key_leaves(seeded):
    # ts_gt is LM_NONE on the first part's row groups, LM_ALL on the third's: those row groups stay, with the key constant
    e, parts, _ = seeded
    keys = [KEYS["ts_gt"]]
    got, st = _run(e, "bk", keys)
    assert st["row_groups_pruned"] == 0
    assert rows_of(got, [keys[0].Name()]) == [(False,), (True,)]


def test_routing_without_the_boolean_key_is_unchanged(seeded, monkeypatch):
    # the plain Distinct(labels.a, labels.b) keeps going to the tile kernel (nullable keys), every row group of it; the
    # same Distinct with a boolean key stays in k_scan, where the tile kernel switched off sends the plain one too
    e, parts, _ = seeded
    got, st = _run(e, "bk", [A, B])
    assert rows_of(got, ["labels.a", "labels.b"]) == ref.distinct_rows(parts, [A, B])
    assert st["row_groups_tiles"] + st["row_groups_runs"] == st["row_groups"] - st["row_groups_pruned"] > 0
    got, st_b = _run(e, "bk", [A, B, KEYS["int_gt"]])
    assert st_b["row_groups_runs"] == 0 and st_b["row_groups_tiles"] == 0 and st_b["row_groups_prefix"] == 0
    monkeypatch.setenv("FROSTGPU_NO_TILE", "1")
    monkeypatch.setenv("FROSTGPU_NO_RUNS", "1")
    got, st_off = _run(e, "bk", [A, B])
    assert rows_of(got, ["labels.a", "labels.b"]) == ref.distinct_rows(parts, [A, B])
    assert st_off["row_groups_tiles"] == st_off["row_groups_runs"] == 0


def test_prepared_plans_cache_and_keep_their_literals(seeded):
    e, parts, _ = seeded
    lib = _lib.load()
    scans = [GPUScan(e, "bk", None, _lib.PLAN_DISTINCT, [A, V.Gt(L(lit))], []) for lit in (0, 1)]
    prepared = [s.prepare() for s in scans]
    try:
        for (q, _), lit in zip(prepared, (0, 1)):
            keys = [A, V.Gt(L(lit))]
            exp = ref.distinct_rows(parts, keys)
            for _ in range(2):  # the second Execute takes the cached path
                res = C.c_void_p()
                _lib.check(lib.fgpu_query_execute(e.handle, q, e.table_watermark("bk"), C.byref(res)))
                try:
                    assert rows_of(list(e.drain(res)), [k.Name() for k in keys]) == exp
                finally:
                    lib.fgpu_result_free(res)
    finally:
        for q, keep in prepared:
            lib.fgpu_query_free(q)


@pytest.mark.parametrize("keys", [[A, B, KEYS["int_gt"]], [N, KEYS["dict_eq"]]], ids=["dense", "hash"])
def test_multirank_collective_equals_single_context(seeded, keys):
    """Two contexts on one GPU (two ranks), each with a share of the parts and the same preloaded dictionaries, run
    the collective Execute the way tests/test_gpu_multirank.py's ranks do (every push before the first wait); each
    must end with the single-context result.  The ranks hold 2 and 1 parts, so their hash tables differ in size."""
    from frostdb_b200.store import comm_setup
    e1, parts, bufs = seeded
    lib = _lib.load()
    names = [k.Name() for k in keys]
    single, _ = _run(e1, "bk", keys)
    assert rows_of(single, names) == _expected(parts, keys)
    engines = [GPUEngine(0), GPUEngine(0)]
    prepared, pend, opened = [], [], False
    try:
        for e, sh in zip(engines, (bufs[0::2], bufs[1::2])):
            for col, card in (("labels.a", 6), ("labels.b", 3)):
                e.dict_preload("mr", col, [v.encode() for v in label_values(card)])
            for b in sh:
                e.put_parquet("mr", b)
        comm_setup(engines, slot_bytes=16 << 20)
        opened = True
        scans = [GPUScan(e, "mr", None, _lib.PLAN_DISTINCT, keys, []) for e in engines]
        prepared = [s.prepare() for s in scans]
        for rep in range(2):  # compiled plan, then the cached one
            pend = [e.execute_collective_begin(p[0], e.table_watermark("mr")) for e, p in zip(engines, prepared)]
            for r, e in enumerate(engines):
                e.execute_collective_end(pend[r])
                got = list(e.drain(pend[r]))
                assert rows_of(got, names) == rows_of(single, names), (r, rep)
            for res in pend:
                lib.fgpu_result_free(res)
            pend = []
    finally:
        for res in pend:
            lib.fgpu_result_free(res)
        for q, _ in prepared:
            lib.fgpu_query_free(q)
        for e in engines:
            if opened:
                e.comm_close()
            e.close()


def _refusal(e, **kw):
    with pytest.raises(_lib.FrostGPUError) as ei:
        _run(e, "bk", **kw)
    return ei.value.code, ei.value.msg


def test_refusals_match_the_filter(seeded):
    e, _, _ = seeded
    as_key = _refusal(e, keys=[A, V.Eq(L("x"))])
    as_filter = _refusal(e, keys=[A], filt=V.Eq(L("x")))
    assert as_key == as_filter == (_lib.FGPU_ERR_UNSUPPORTED, "numeric column compared with a string literal")
    filt = lp.Or(*[A.Eq(L(f"v{i:06d}")) for i in range(20)])
    key = lp.Or(*[B.Eq(L(f"v{i:06d}")) for i in range(13)])
    assert _refusal(e, keys=[A, key], filt=filt) == (_lib.FGPU_ERR_UNSUPPORTED, "too many predicate leaves")
    _run(e, "bk", [A, lp.Or(*[B.Eq(L(f"v{i:06d}")) for i in range(12)])], filt)  # 32 leaves in all: accepted
    assert _refusal(e, keys=[A, V.Gt(L(0))], kind=_lib.PLAN_AGGREGATE, aggs=[lp.Count(V)]) == (
        _lib.FGPU_ERR_UNSUPPORTED, "this group-by expression is not supported on the GPU path")
