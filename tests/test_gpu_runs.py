"""Sorted-run kernel (k_runs) and statistics pruning against the oracle, and against the general scan
kernel with both switched off (FROSTGPU_NO_RUNS / FROSTGPU_NO_PRUNE): the three ways to run a query must
give identical records."""
import ctypes as C
import os

import numpy as np
import pyarrow as pa
import pytest

from frostdb_b200 import _lib
from frostdb_b200 import dynparquet as dp
from frostdb_b200 import logicalplan as lp
from frostdb_b200.physicalplan import GPUScan
from tests.test_gpu_parity import Pair, assert_same
from tests.util import label_values, rows_of

pytestmark = pytest.mark.gpu


def sorted_columns(n, seed, *, t0=0, cards=(5, 23), run_scale=1.0, third=None, with_float=False):
    """Non-null label columns a, b (and optionally c) whose sort leaves runs of very different lengths."""
    rng = np.random.default_rng(seed)
    cols = {
        "example_type": (np.zeros(n, np.int32), ["cpu"]),
        "stacktrace": (rng.integers(0, 11, n).astype(np.int32), [f"stack{i:02d}" for i in range(11)]),
        "timestamp": t0 + np.arange(n, dtype=np.int64),
        "value": rng.integers(-500, 1000, n).astype(np.int64),
    }
    # skewed group sizes: some (a, b) groups hold a handful of rows, others thousands
    w = rng.random(cards[0] * cards[1]) ** (4.0 * run_scale)
    g = rng.choice(cards[0] * cards[1], size=n, p=w / w.sum())
    cols["labels.a"] = ((g // cards[1]).astype(np.int32), label_values(cards[0]))
    cols["labels.b"] = ((g % cards[1]).astype(np.int32), label_values(cards[1]))
    if third:
        cols["labels.c"] = (rng.integers(0, third, n).astype(np.int32), label_values(third))
    if with_float:
        cols["floatvalue"] = pa.array((rng.integers(-10**6, 10**6, n).astype(np.float64)) / 997.0)
    return cols


@pytest.fixture()
def pair(store):
    made = []

    def make(name, schema=None):
        p = Pair(store, name, schema or dp.SampleDefinition())
        made.append(p)
        return p
    yield make
    for p in made:
        p.close()
    for k in ("FROSTGPU_NO_RUNS", "FROSTGPU_NO_PRUNE"):
        os.environ.pop(k, None)


def run3(p, build, float_cols=()):
    """default path, no sorted-run kernel, no pruning: all equal to the oracle"""
    got, exp = p.run(build)
    assert_same(got, exp, float_cols)
    for env in ({"FROSTGPU_NO_RUNS": "1"}, {"FROSTGPU_NO_PRUNE": "1"}, {"FROSTGPU_NO_RUNS": "1", "FROSTGPU_NO_PRUNE": "1"}):
        os.environ.update(env)
        try:
            got2, _ = p.run(build)
        finally:
            for k in env:
                os.environ.pop(k)
        assert_same(got2, exp, float_cols)
    return got


def scan_stats(p, filt, aggs, groups):
    eng = p.store.engine
    scan = GPUScan(eng, p.name, filt, _lib.PLAN_AGGREGATE, groups, aggs)
    q, keep = scan.prepare()
    lib = _lib.load()
    res = C.c_void_p()
    _lib.check(lib.fgpu_query_execute(eng.handle, q, eng.table_watermark(p.name), C.byref(res)))
    st = eng.stats(res)
    lib.fgpu_result_free(res)
    lib.fgpu_query_free(q)
    return st


AGGS = [lp.Sum(lp.Col("value")), lp.Count(lp.Col("value"))]
KEYS = [lp.Col("labels.a"), lp.Col("labels.b")]


@pytest.mark.parametrize("rows,rg", [(100_000, 32_768), (33_333, 10_007), (4_099, 4_099)])
def test_sorted_parts_group_by_two_keys(pair, rows, rg):
    p = pair("runs2")
    for i in range(3):
        p.insert(sorted_columns(rows, 100 + i, t0=i * rows), row_group_size=rg, data_page_size=16_384)
    run3(p, lambda q: q.Aggregate(AGGS, KEYS))
    st = scan_stats(p, None, AGGS, KEYS)
    assert st["row_groups_runs"] == st["row_groups"] > 0  # every row group of a sorted part takes the run kernel
    run3(p, lambda q: q.Aggregate([lp.Count(lp.Col("value"))], KEYS))
    run3(p, lambda q: q.Aggregate([lp.Sum(lp.Col("value")), lp.Sum(lp.Col("timestamp"))], [lp.Col("labels.a")]))
    run3(p, lambda q: q.Aggregate(AGGS, []))


def test_time_range_filters_prune_and_split(pair):
    p = pair("runs_prune")
    n = 50_000
    for i in range(6):
        p.insert(sorted_columns(n, 200 + i, t0=i * n), row_group_size=20_000)
    ts = lp.Col("timestamp")
    cases = [
        lp.And(ts.GtEq(lp.Literal(n + 17)), ts.Lt(lp.Literal(4 * n + 5))),   # parts 0 and 5 out, 2 and 3 fully inside
        lp.And(ts.GtEq(lp.Literal(2 * n)), ts.Lt(lp.Literal(4 * n))),        # exact part boundaries
        ts.Lt(lp.Literal(10)),                                               # ten rows of the first part
        ts.Gt(lp.Literal(10 * n)),                                           # nothing
        ts.GtEq(lp.Literal(0)),                                              # everything, decided by statistics alone
        lp.And(ts.GtEq(lp.Literal(n // 2)), lp.Col("value").Gt(lp.Literal(250))),  # two leaves, two columns
        lp.And(ts.LtEq(lp.Literal(5 * n)), lp.Col("value").GtEq(lp.Literal(-500))),  # second leaf always true
        lp.And(lp.Col("value").Gt(lp.Literal(100)), lp.Col("value").LtEq(lp.Literal(700))),  # filter column == aggregate input
        ts.NotEq(lp.Literal(3 * n)),                                         # negated range: general kernel, statistics still apply
        lp.Or(ts.Lt(lp.Literal(n)), ts.GtEq(lp.Literal(5 * n))),             # disjunction: no row group is dropped
    ]
    for f in cases:
        try:
            run3(p, lambda q: q.Filter(f).Aggregate(AGGS, KEYS))
            run3(p, lambda q: q.Filter(f).Aggregate([lp.Count(lp.Col("value"))], [lp.Col("labels.a")]))
        except AssertionError as e:
            raise AssertionError(f"filter {f.Name()}: {e}") from e
    st = scan_stats(p, cases[0], AGGS, KEYS)
    assert st["row_groups_pruned"] > 0 and st["row_groups_runs"] > 0
    assert st["row_groups_pruned"] + st["row_groups"] == 6 * 3
    st = scan_stats(p, cases[3], AGGS, KEYS)
    assert st["row_groups"] == 0 and st["rows_selected"] == 0
    # rows plans keep their order when row groups are dropped
    got, exp = p.run(lambda q: q.Filter(cases[0]).Project(lp.Col("timestamp"), lp.Col("value"), lp.Col("labels.b")))
    names = ["timestamp", "value", "labels.b"]
    assert rows_of(got, names) == rows_of(exp, names) and len(rows_of(got, names)) > 0


def test_short_runs_and_three_keys(pair):
    p = pair("runs_short")
    # third sort key with a few values: runs of labels.c are often shorter than a warp
    p.insert(sorted_columns(60_000, 301, cards=(3, 7), third=4), row_group_size=25_000)
    p.insert(sorted_columns(60_000, 302, cards=(3, 7), third=40, run_scale=0.2, t0=60_000), row_group_size=25_000)
    keys3 = KEYS + [lp.Col("labels.c")]
    run3(p, lambda q: q.Aggregate(AGGS, keys3))
    f = lp.And(lp.Col("timestamp").GtEq(lp.Literal(1000)), lp.Col("timestamp").Lt(lp.Literal(100_000)))
    run3(p, lambda q: q.Filter(f).Aggregate(AGGS, keys3))
    run3(p, lambda q: q.Filter(f).Aggregate(AGGS, [lp.Col("labels.c")]))  # not a sort prefix: long bit-packed runs


def test_unsorted_and_nullable_parts_fall_back(pair):
    p = pair("runs_mixed")
    p.insert(sorted_columns(40_000, 401), row_group_size=16_000)
    cols = sorted_columns(40_000, 402, t0=40_000)
    p.insert(cols, sort=False, row_group_size=16_000)                # arrival order: bit-packed key columns
    cols = sorted_columns(40_000, 403, t0=80_000)
    idx = cols["labels.b"][0].copy()
    idx[::7] = -1                                                    # NULL keys
    cols["labels.b"] = (idx, cols["labels.b"][1])
    p.insert(cols, row_group_size=16_000)
    f = lp.Col("timestamp").GtEq(lp.Literal(20_000))
    run3(p, lambda q: q.Filter(f).Aggregate(AGGS, KEYS))
    st = scan_stats(p, f, AGGS, KEYS)
    assert 0 < st["row_groups_runs"] < st["row_groups"]


def test_without_statistics_nothing_is_pruned(pair):
    p = pair("runs_nostats")
    for i in range(2):
        p.insert(sorted_columns(30_000, 500 + i, t0=i * 30_000), row_group_size=10_000, write_statistics=False)
    f = lp.Col("timestamp").Lt(lp.Literal(15_000))
    run3(p, lambda q: q.Filter(f).Aggregate(AGGS, KEYS))
    st = scan_stats(p, f, AGGS, KEYS)
    assert st["row_groups_pruned"] == 0


def test_min_max_and_float_aggregates_on_sorted_parts(pair):
    p = pair("runs_minmax", dp.SampleDefinitionWithFloat())
    n = 70_001
    for i in range(3):
        p.insert(sorted_columns(n, 600 + i, t0=i * n, with_float=True), row_group_size=30_000)
    v, fv, ts = lp.Col("value"), lp.Col("floatvalue"), lp.Col("timestamp")
    f = lp.And(ts.GtEq(lp.Literal(n // 3)), ts.Lt(lp.Literal(2 * n + 11)))
    cases = [
        ([lp.Sum(v), lp.Min(v)], ()), ([lp.Max(v), lp.Min(v), lp.Count(v)], ()), ([lp.Min(ts), lp.Max(ts)], ()),
        ([lp.Sum(fv), lp.Max(v)], ("sum(floatvalue)",)), ([lp.Min(fv), lp.Max(fv)], ()), ([lp.Sum(fv), lp.Sum(v)], ("sum(floatvalue)",)),
        ([lp.Sum(v), lp.Min(v), lp.Max(v), lp.Count(v)], ()), ([lp.Sum(fv), lp.Min(ts), lp.Max(v)], ("sum(floatvalue)",)),
    ]
    for aggs, fcols in cases:
        for flt in (None, f):
            build = (lambda q: q.Filter(flt).Aggregate(aggs, KEYS)) if flt is not None else (lambda q: q.Aggregate(aggs, KEYS))
            try:
                run3(p, build, fcols)
            except AssertionError as e:
                raise AssertionError(f"{[a.Name() for a in aggs]} filter={flt is not None}: {e}") from e
    st = scan_stats(p, f, [lp.Min(fv), lp.Sum(v)], KEYS)
    assert st["row_groups_runs"] == st["row_groups"] > 0


def test_filter_only_plans_take_path(pair):
    """TableScan -> Filter -> Projection(PLAIN columns): the ordered take kernels against the oracle and
    against k_rows (FROSTGPU_NO_TAKE), over selectivities from nothing to everything."""
    p = pair("take", dp.SampleDefinitionWithFloat())
    n = 41_003
    for i in range(4):
        p.insert(sorted_columns(n, 800 + i, t0=i * n, with_float=True), row_group_size=15_000)
    ts, v, fv = lp.Col("timestamp"), lp.Col("value"), lp.Col("floatvalue")
    filters = [
        ts.Lt(lp.Literal(int(0.001 * 4 * n))), ts.Lt(lp.Literal(2 * n + 7)), ts.GtEq(lp.Literal(0)), ts.Gt(lp.Literal(9 * n)),
        v.Lt(lp.Literal(-499)), v.Lt(lp.Literal(250)), v.GtEq(lp.Literal(-500)),
        lp.And(lp.And(ts.GtEq(lp.Literal(n // 2)), ts.Lt(lp.Literal(3 * n))), v.Gt(lp.Literal(900))),
        lp.And(ts.LtEq(lp.Literal(10 * n)), v.Eq(lp.Literal(77))),
    ]
    names = ["timestamp", "value", "floatvalue"]
    for f in filters:
        for proj in ([ts, v], [v], [fv, ts, v]):
            cols = [e.Name() for e in proj]
            got, exp = p.run(lambda q: q.Filter(f).Project(*proj))
            os.environ["FROSTGPU_NO_TAKE"] = "1"
            try:
                got2, _ = p.run(lambda q: q.Filter(f).Project(*proj))
            finally:
                os.environ.pop("FROSTGPU_NO_TAKE")
            # order-preserving: compare WITHOUT sorting
            def flat(batches):
                out = []
                for b in batches:
                    if b.num_rows == 0:
                        continue  # (an empty selection: no record, or an empty one)
                    out.extend(zip(*[b.column(b.schema.get_field_index(c)).to_pylist() for c in cols]))
                return out
            assert flat(got) == flat(exp) == flat(got2), f"{f.Name()} -> {cols}"


def test_string_equality_prunes_row_groups_by_bounds(pair):
    p = pair("runs_strprune")
    n = 60_000
    for i in range(3):
        p.insert(sorted_columns(n, 900 + i, t0=i * n, cards=(6, 9)), row_group_size=7_000)
    a, b = lp.Col("labels.a"), lp.Col("labels.b")
    for f in (a.Eq(lp.Literal("v000002")), a.Eq(lp.Literal("v000009")), a.Eq(lp.Literal("")), a.NotEq(lp.Literal("v000002")),
              lp.And(a.Eq(lp.Literal("v000004")), lp.Col("timestamp").Lt(lp.Literal(2 * n))),
              lp.Or(a.Eq(lp.Literal("v000000")), b.Eq(lp.Literal("v000003")))):
        try:
            run3(p, lambda q: q.Filter(f).Aggregate(AGGS, KEYS))
        except AssertionError as e:
            raise AssertionError(f"filter {f.Name()}: {e}") from e
    st = scan_stats(p, a.Eq(lp.Literal("v000002")), AGGS, KEYS)
    assert 0 < st["row_groups_pruned"] < 27 and st["rows_selected"] > 0
    st = scan_stats(p, a.Eq(lp.Literal("v000009")), AGGS, KEYS)   # beyond every chunk's maximum
    assert st["row_groups"] == 0


def test_nullable_sorted_keys_take_the_run_kernel(pair):
    """NULL keys sort first (compaction order): levels and indices are both run-length, the host merges them
    into one directory in row space and the row groups stay with k_runs."""
    p = pair("runs_nullkeys")
    n = 50_000
    for i in range(3):
        cols = sorted_columns(n, 950 + i, t0=i * n, cards=(4, 17))
        rng = np.random.default_rng(i)
        for name, pnull in (("labels.a", 0.15), ("labels.b", 0.3)):
            idx = cols[name][0].copy()
            idx[rng.random(n) < pnull] = -1
            cols[name] = (idx, cols[name][1])
        p.insert(cols, row_group_size=21_000)
    f = lp.And(lp.Col("timestamp").GtEq(lp.Literal(n // 4)), lp.Col("timestamp").Lt(lp.Literal(2 * n + 5)))
    for flt in (None, f):
        build = (lambda q: q.Filter(flt).Aggregate(AGGS, KEYS)) if flt is not None else (lambda q: q.Aggregate(AGGS, KEYS))
        run3(p, build)
        build1 = (lambda q: q.Filter(flt).Aggregate(AGGS, [lp.Col("labels.a")])) if flt is not None else (lambda q: q.Aggregate(AGGS, [lp.Col("labels.a")]))
        run3(p, build1)
    st = scan_stats(p, None, AGGS, KEYS)
    assert st["row_groups_runs"] == st["row_groups"] > 0


def test_dictionary_leaves_evaluated_once_per_run(pair):
    """label == / != / regex / contains / == NULL on run-length columns run inside k_runs (one result per run)."""
    p = pair("runs_dictleaf")
    n = 45_000
    for i in range(3):
        cols = sorted_columns(n, 970 + i, t0=i * n, cards=(6, 19), third=5)
        idx = cols["labels.b"][0].copy()
        idx[np.random.default_rng(i).random(n) < 0.2] = -1          # nullable second key
        cols["labels.b"] = (idx, cols["labels.b"][1])
        p.insert(cols, row_group_size=16_000)
    a, b, cc, ts = lp.Col("labels.a"), lp.Col("labels.b"), lp.Col("labels.c"), lp.Col("timestamp")
    rng = lp.And(ts.GtEq(lp.Literal(n // 3)), ts.Lt(lp.Literal(2 * n + 9)))
    filters = [
        a.Eq(lp.Literal("v000003")), a.NotEq(lp.Literal("v000003")), b.Eq(lp.Literal(None)), b.NotEq(lp.Literal(None)),
        b.RegexMatch("v00000[2-5]$"), b.Contains("01"), lp.And(a.Eq(lp.Literal("v000001")), b.NotEq(lp.Literal("v000004"))),
        lp.And(rng, a.Eq(lp.Literal("v000002"))), lp.And(lp.And(rng, b.RegexNotMatch("v00001")), lp.Col("value").Gt(lp.Literal(0))),
        lp.And(a.Eq(lp.Literal("v000004")), lp.Col("labels.zz").Eq(lp.Literal(""))),   # absent column: decided everywhere
        lp.And(a.Eq(lp.Literal("v000000")), cc.Eq(lp.Literal("v000001"))),             # labels.c is not run-length: general kernel
    ]
    for f in filters:
        try:
            run3(p, lambda q: q.Filter(f).Aggregate(AGGS, KEYS))
            run3(p, lambda q: q.Filter(f).Aggregate([lp.Max(lp.Col("value")), lp.Count(lp.Col("value"))], [b]))
        except AssertionError as e:
            raise AssertionError(f"filter {f.Name()}: {e}") from e
    st = scan_stats(p, filters[7], AGGS, KEYS)
    assert st["row_groups_runs"] == st["row_groups"] > 0 and st["rows_selected"] > 0
    st = scan_stats(p, filters[4], AGGS, KEYS)
    assert st["row_groups_runs"] == st["row_groups"] > 0


def test_prepared_query_reexecuted_and_invalidated(pair):
    """A prepared query keeps its compiled plan while the table is unchanged; a new part, a dropped part or a new
    read transaction must recompile.  Every execution equals a freshly prepared one."""
    p = pair("plan_cache")
    n = 30_000
    eng, lib = p.store.engine, _lib.load()
    f = lp.And(lp.Col("timestamp").GtEq(lp.Literal(n // 2)), lp.Col("labels.a").NotEq(lp.Literal("v000001")))
    names = ["labels.a", "labels.b", "sum(value)", "count(value)"]

    def execute(q):
        res = C.c_void_p()
        _lib.check(lib.fgpu_query_execute(eng.handle, q, eng.table_watermark(p.name), C.byref(res)))
        out = list(eng.drain(res))
        lib.fgpu_result_free(res)
        return rows_of(out, names)

    def fresh():
        q, keep = GPUScan(eng, p.name, f, _lib.PLAN_AGGREGATE, KEYS, AGGS).prepare()
        try:
            return execute(q)
        finally:
            lib.fgpu_query_free(q)

    p.insert(sorted_columns(n, 990, t0=0), row_group_size=11_000)
    p.insert(sorted_columns(n, 991, t0=n), sort=False)
    q, keep = GPUScan(eng, p.name, f, _lib.PLAN_AGGREGATE, KEYS, AGGS).prepare()
    try:
        first = execute(q)
        assert first == execute(q) == execute(q) == fresh() and len(first) > 0
        got, exp = p.run(lambda b: b.Filter(f).Aggregate(AGGS, KEYS))
        assert rows_of(got, names) == rows_of(exp, names) == first
        p.insert(sorted_columns(n, 992, t0=2 * n, cards=(7, 29)), row_group_size=9_000)   # new part, new dictionary entries
        second = execute(q)
        assert second == execute(q) == fresh() and second != first
        got, exp = p.run(lambda b: b.Filter(f).Aggregate(AGGS, KEYS))
        assert rows_of(got, names) == rows_of(exp, names) == second
        eng.drop_part(p.name, 2)
        assert execute(q) == first
    finally:
        lib.fgpu_query_free(q)


def test_global_max_skips_row_groups_below_the_running_maximum(pair):
    """AggFuncPushDown + MaxAgg (logicalplan/optimize.go:166-193, expr/filter.go:156-207): Max(column) without group-by
    and filter only reads the row groups whose chunk maximum exceeds the largest one seen before them."""
    p = pair("maxagg")
    n = 40_000
    for i in range(4):
        p.insert(sorted_columns(n, 300 + i, t0=(3 - i) * n), row_group_size=10_000)   # later parts hold EARLIER timestamps
    run3(p, lambda q: q.Aggregate([lp.Max(lp.Col("timestamp"))], []))
    st = scan_stats(p, None, [lp.Max(lp.Col("timestamp"))], [])
    assert st["row_groups_pruned"] >= 12 and st["row_groups"] <= 4   # only the first part's row groups raise the maximum
    run3(p, lambda q: q.Aggregate([lp.Max(lp.Col("value"))], []))
    run3(p, lambda q: q.Aggregate([lp.Min(lp.Col("timestamp"))], []))    # no push-down for Min


def test_locally_dense_runs_leave_the_staged_directory_window(pair):
    """k_runs_tma stages 128 directory entries per key and 4096-row tile; a tile that holds more runs than that walks
    the rest of the directory in global memory (cursor_global).  Row groups whose runs average >= 32 rows qualify for
    the kernel, so: a row group whose first rows change group every 2-3 rows while the rest is a few huge groups."""
    n = 200_000
    rng = np.random.default_rng(77)
    dense = 9_000                                  # rows with short runs (they sort first: small ids)
    a = np.empty(n, np.int32)
    b = np.empty(n, np.int32)
    a[:dense] = 0
    # runs of 8-12 rows (a Parquet writer only run-length encodes 8 repeats and more; shorter ones would leave the
    # column bit-packed and with it the sorted-run kernel): ~400 runs in the first 4096-row tile
    reps = rng.integers(8, 13, 2_000)
    b[:dense] = np.repeat(np.arange(2_000, dtype=np.int32), reps)[:dense]
    a[dense:] = np.sort(rng.integers(1, 4, n - dense)).astype(np.int32)
    b[dense:] = 2_000 + rng.integers(0, 3, n - dense).astype(np.int32)
    cols = {
        "example_type": (np.zeros(n, np.int32), ["cpu"]),
        "stacktrace": (rng.integers(0, 5, n).astype(np.int32), [f"stack{i:02d}" for i in range(5)]),
        "timestamp": np.arange(n, dtype=np.int64),
        "value": rng.integers(-1000, 1000, n).astype(np.int64),
        "labels.a": (a, label_values(4)),
        "labels.b": (b, label_values(2_003)),
    }
    p = pair("runs_dense_window")
    p.insert(cols, row_group_size=n, data_page_size=1 << 20)
    ts, val = lp.Col("timestamp"), lp.Col("value")
    run3(p, lambda q: q.Aggregate(AGGS, KEYS))
    st = scan_stats(p, None, AGGS, KEYS)
    assert st["row_groups_runs"] == st["row_groups"] == 1
    run3(p, lambda q: q.Filter(val.Gt(lp.Literal(0))).Aggregate(AGGS, KEYS))                       # row filter: 2048-row tiles... one column
    run3(p, lambda q: q.Filter(lp.And(ts.GtEq(lp.Literal(1_000)), val.LtEq(lp.Literal(500)))).Aggregate(AGGS, KEYS))  # two staged columns
    run3(p, lambda q: q.Filter(lp.Col("labels.b").NotEq(lp.Literal("v000007"))).Aggregate(AGGS, [lp.Col("labels.a")]))  # leaf cursor beyond the window
    run3(p, lambda q: q.Filter(ts.Lt(lp.Literal(3_000))).Aggregate([lp.Sum(val), lp.Min(val), lp.Max(val)], KEYS))        # general reducers


@pytest.mark.parametrize("env", [{"FROSTGPU_RT_TILE": "1024", "FROSTGPU_RT_WARPS": "4", "FROSTGPU_RT_SPAN": "1"},
                                 {"FROSTGPU_RT_TILE": "8192", "FROSTGPU_RT_STAGES": "2", "FROSTGPU_RT_SPAN": "3"},
                                 {"FROSTGPU_RT_TILE": "2048", "FROSTGPU_RT_STAGES": "4", "FROSTGPU_RT_SPAN": "16"}])
def test_tile_ring_and_chunk_shapes_give_the_same_records(pair, env):
    p = pair("runs_shapes")
    for i in range(3):
        p.insert(sorted_columns(70_001, 900 + i, t0=i * 70_001, third=3), row_group_size=33_000)
    os.environ.update(env)
    try:
        ts = lp.Col("timestamp")
        got, exp = p.run(lambda q: q.Aggregate(AGGS, KEYS))
        assert_same(got, exp, ())
        got, exp = p.run(lambda q: q.Filter(lp.And(ts.GtEq(lp.Literal(50_000)), ts.Lt(lp.Literal(150_000)))).Aggregate(AGGS, KEYS + [lp.Col("labels.c")]))
        assert_same(got, exp, ())
        got, exp = p.run(lambda q: q.Filter(lp.Col("value").Lt(lp.Literal(0))).Aggregate([lp.Count(lp.Col("value"))], []))
        assert_same(got, exp, ())
    finally:
        for k in env:
            os.environ.pop(k)


def test_filter_only_plans_with_dictionary_leaves_take_path(pair):
    """cfg 5 with a dict-string predicate: ==, !=, contains, regex and == NULL leaves on dictionary columns (sorted
    and unsorted parts, NULLs in the column, a column missing from one part) — the ordered take kernels over flat
    codes against the oracle and against k_rows (FROSTGPU_NO_TAKE), without sorting the rows."""
    from tests.util import make_columns
    p = pair("take_dict")
    n = 30_011
    p.insert(sorted_columns(n, 810, t0=0, third=5), row_group_size=11_000)
    p.insert(make_columns(n, 811, {"a": (5, 0.0), "b": (23, 0.2), "c": (5, 0.5)}, t0=n), row_group_size=9_000, sort=False)
    p.insert(make_columns(n, 812, {"a": (5, 0.1), "b": (23, 0.0)}, t0=2 * n), row_group_size=30_011)   # no labels.c here
    ts, v = lp.Col("timestamp"), lp.Col("value")
    a, b, c = lp.Col("labels.a"), lp.Col("labels.b"), lp.Col("labels.c")
    filters = [
        a.Eq(lp.Literal("v000002")), b.NotEq(lp.Literal("v000007")), c.Eq(lp.Literal(None)), c.NotEq(lp.Literal(None)),
        b.Contains("0001"), b.RegexMatch("v00000[1-3]"), a.Eq(lp.Literal("nope")),
        lp.And(a.Eq(lp.Literal("v000001")), ts.Lt(lp.Literal(2 * n + 100))),
        lp.And(lp.And(b.NotEq(lp.Literal("v000003")), c.Eq(lp.Literal("v000004"))), v.Gt(lp.Literal(100))),
        lp.And(c.Eq(lp.Literal("")), ts.GtEq(lp.Literal(n))),   # missing column == "": every row of the part without it
    ]
    for f in filters:
        for proj in ([ts, v], [v], [v, c]):  # labels.c: k_rows reads the part without it as NULL
            cols = [e.Name() for e in proj]
            got, exp = p.run(lambda q: q.Filter(f).Project(*proj))
            os.environ["FROSTGPU_NO_TAKE"] = "1"
            try:
                got2, _ = p.run(lambda q: q.Filter(f).Project(*proj))
            finally:
                os.environ.pop("FROSTGPU_NO_TAKE")

            def flat(batches):  # (a record of a part without labels.c may leave that column out: NULL)
                out = []
                for bt in batches:
                    if bt.num_rows:
                        idx = [bt.schema.get_field_index(cn) for cn in cols]
                        out.extend(zip(*[bt.column(i).to_pylist() if i >= 0 else [None] * bt.num_rows for i in idx]))
                return out
            assert flat(got) == flat(exp) == flat(got2), f"{f.Name()} -> {cols}"


def test_bloom_filters_prune_equality_leaves(store):
    """Chunks with split-block bloom filters (what parquet-go writes for FrostDB's sorting columns): `x == v` with v
    inside [min, max] but not in the chunk drops the row group before anything is uploaded; under a disjunction the row
    group stays and the leaf is false on all of its rows; values that are there are found."""
    from tests import bloom_file as bf
    eng = store.engine
    rng = np.random.default_rng(11)
    parts = []
    for i in range(3):
        xs = [int(v) for v in rng.integers(0, 100_000, 5_000)]
        ys = [int(v) for v in rng.integers(0, 10, 5_000)]
        parts.append((xs, ys))
        eng.put_parquet("bloomy", bf.write_int64_file({"x": xs, "y": ys}))
    try:
        x, y = lp.Col("x"), lp.Col("y")
        all_x = [v for xs, _ in parts for v in xs]
        absent = None
        for v in range(50_000, 50_400):  # a value no part holds and every part's filter rejects
            if v in all_x:
                continue
            if all(not bf.sbbf_check(_bits(xs), bf.xxh64(v.to_bytes(8, "little", signed=True))) for xs, _ in parts):
                absent = v
                break
        assert absent is not None
        def run(filt, aggs=None):
            scan = GPUScan(eng, "bloomy", filt, _lib.PLAN_AGGREGATE, [], aggs or [lp.Count(x), lp.Sum(y)])
            q, keep = scan.prepare()
            lib = _lib.load()
            res = C.c_void_p()
            _lib.check(lib.fgpu_query_execute(eng.handle, q, eng.table_watermark("bloomy"), C.byref(res)))
            st = eng.stats(res)
            rows = rows_of(list(eng.drain(res)))
            lib.fgpu_result_free(res)
            lib.fgpu_query_free(q)
            return st, rows
        st, rows = run(x.Eq(lp.Literal(absent)))
        assert st["row_groups_pruned"] == 3 and st["row_groups"] == 0 and rows == []
        present = parts[1][0][17]
        st, rows = run(x.Eq(lp.Literal(present)))
        exp_n = sum(xs.count(present) for xs, _ in parts)
        exp_s = sum(yv for xs, ys in parts for xv, yv in zip(xs, ys) if xv == present)
        assert rows == [(exp_n, exp_s)]
        assert st["row_groups_pruned"] >= 1  # the parts whose filters do not know the value
        st, rows = run(lp.Or(x.Eq(lp.Literal(absent)), y.Eq(lp.Literal(3))))
        exp_n = sum(1 for _, ys in parts for yv in ys if yv == 3)
        assert st["row_groups_pruned"] == 0 and rows == [(exp_n, 3 * exp_n)]
    finally:
        eng.drop_table("bloomy")


def _bits(xs):
    from tests import bloom_file as bf
    n_bytes = max(32, ((len(xs) * 10 // 8) + 31) // 32 * 32)
    bits = bytearray(n_bytes)
    for v in xs:
        bf.sbbf_insert(bits, bf.xxh64(v.to_bytes(8, "little", signed=True)))
    return bytes(bits)
