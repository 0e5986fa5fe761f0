"""Prefix path of the sorted-run scan (k_runs_prefix): all-pass row groups whose stored aggregates are all Sum(int64)
are answered from the key run directories and exclusive prefix sums of the Sum inputs.  Every case is compared with the
oracle and with the prefix path, the sorted-run kernels and pruning switched off (FROSTGPU_NO_PREFIX / _NO_RUNS /
_NO_PRUNE), and the cases assert which row groups took the prefix path."""
import ctypes as C
import os

import numpy as np
import pytest

from frostdb_b200 import _lib
from frostdb_b200 import dynparquet as dp
from frostdb_b200 import logicalplan as lp
from frostdb_b200.physicalplan import GPUScan
from tests.test_gpu_parity import assert_same
from tests.test_gpu_runs import AGGS, KEYS, pair, run3, scan_stats, sorted_columns  # noqa: F401  (pair: fixture)
from tests.test_gpu_runs_narrow import EXTREMES, part_with_chunks
from tests.util import label_values, rows_of

pytestmark = pytest.mark.gpu

ts, val = lp.Col("timestamp"), lp.Col("value")


def with_env(env, fn):
    os.environ.update(env)
    try:
        return fn()
    finally:
        for k in env:
            os.environ.pop(k)


def run4(p, build, float_cols=()):
    """run3 (oracle, no sorted-run kernels, no pruning) and the same without the prefix path"""
    got = run3(p, build, float_cols)
    got2, exp = with_env({"FROSTGPU_NO_PREFIX": "1"}, lambda: p.run(build))
    assert_same(got2, exp, float_cols)
    return got


def prefix_stats(p, filt, aggs, keys):
    """stats with the prefix path, and rows_selected must equal the one without it"""
    st = scan_stats(p, filt, aggs, keys)
    off = with_env({"FROSTGPU_NO_PREFIX": "1"}, lambda: scan_stats(p, filt, aggs, keys))
    assert off["row_groups_prefix"] == 0 and off["row_groups_runs"] == st["row_groups_runs"]
    assert st["rows_selected"] == off["rows_selected"]
    return st


def check_shapes(p, filt, keysets):
    for keys in keysets:
        for aggs in (AGGS, [lp.Sum(val), lp.Sum(ts)], [lp.Count(val)]):
            build = (lambda q: q.Filter(filt).Aggregate(aggs, keys)) if filt is not None else (lambda q: q.Aggregate(aggs, keys))
            try:
                run4(p, build)
            except AssertionError as e:
                raise AssertionError(f"keys {[k.Name() for k in keys]} aggs {[a.Name() for a in aggs]}: {e}") from e


def test_keys_aggregates_and_mixed_launches(pair):
    p = pair("prefix_shapes")
    n = 40_013
    for i in range(3):  # row groups of 10 007 rows: not a multiple of any window
        p.insert(sorted_columns(n, 1100 + i, t0=i * n, cards=(3, 5), third=3), row_group_size=10_007)
    p.insert(sorted_columns(4_099, 1199, t0=3 * n, cards=(2, 3)), row_group_size=1_000)  # row groups of a few hundred rows
    keysets = [[], KEYS[:1], KEYS, KEYS + [lp.Col("labels.c")]]
    check_shapes(p, None, keysets)
    st = prefix_stats(p, None, AGGS, KEYS + [lp.Col("labels.c")])
    assert st["row_groups_prefix"] >= 12  # (at least the 10 007-row ones: runs average >= 64 rows there)
    st = prefix_stats(p, None, [lp.Count(val)], [])
    assert st["row_groups_prefix"] == st["row_groups"] > 0
    # a time window that leaves all-pass row groups and row groups filtered row by row in one Execute
    f = lp.And(ts.GtEq(lp.Literal(5_000)), ts.Lt(lp.Literal(2 * n + 3_333)))
    check_shapes(p, f, keysets)
    st = prefix_stats(p, f, AGGS, KEYS)
    assert 0 < st["row_groups_prefix"] < st["row_groups_runs"] == st["row_groups"]


def test_nullable_run_length_keys(pair):
    p = pair("prefix_nullkeys")
    n = 50_000
    for i in range(2):
        cols = sorted_columns(n, 1200 + i, t0=i * n, cards=(4, 9))
        rng = np.random.default_rng(i)
        for name, pnull in (("labels.a", 0.15), ("labels.b", 0.3)):
            idx = cols[name][0].copy()
            idx[rng.random(n) < pnull] = -1
            cols[name] = (idx, cols[name][1])
        p.insert(cols, row_group_size=21_000)
    check_shapes(p, None, [KEYS, KEYS[:1]])
    st = prefix_stats(p, None, AGGS, KEYS)
    assert st["row_groups_prefix"] == st["row_groups"] > 0


def test_locally_dense_runs(pair):
    """A row group whose first rows change group every 8-12 rows: windows there hold many more run starts than lanes."""
    n = 200_000
    rng = np.random.default_rng(78)
    dense = 9_000
    a = np.empty(n, np.int32)
    b = np.empty(n, np.int32)
    a[:dense] = 0
    b[:dense] = np.repeat(np.arange(2_000, dtype=np.int32), rng.integers(8, 13, 2_000))[:dense]
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
    p = pair("prefix_dense")
    p.insert(cols, row_group_size=n, data_page_size=1 << 20)
    check_shapes(p, None, [KEYS, KEYS[:1], [lp.Col("labels.b")]])
    st = prefix_stats(p, None, AGGS, KEYS)
    assert st["row_groups_prefix"] == st["row_groups"] == 1


def test_wrapping_sums_at_the_ends_of_int64(pair):
    p = pair("prefix_extremes")
    p.insert(part_with_chunks(EXTREMES, 13), row_group_size=6_000)  # one chunk needs all 64 bits
    run4(p, lambda q: q.Aggregate(AGGS, KEYS))
    run4(p, lambda q: q.Aggregate([lp.Sum(val)], []))
    run4(p, lambda q: q.Aggregate([lp.Sum(val), lp.Sum(ts), lp.Count(val)], KEYS[:1]))
    st = prefix_stats(p, None, AGGS, KEYS)
    assert st["row_groups_prefix"] == st["row_groups"] == len(EXTREMES)


def test_without_statistics_nothing_is_all_pass(pair):
    p = pair("prefix_nostats")
    for i in range(2):
        p.insert(sorted_columns(30_000, 1300 + i, t0=i * 30_000, cards=(3, 5)), row_group_size=10_000, write_statistics=False)
    f = ts.GtEq(lp.Literal(0))
    run4(p, lambda q: q.Filter(f).Aggregate(AGGS, KEYS))
    st = prefix_stats(p, f, AGGS, KEYS)
    assert st["row_groups_prefix"] == 0 and st["row_groups_runs"] == st["row_groups"] > 0


def test_min_max_and_float_sums_stay_with_the_run_kernel(pair):
    p = pair("prefix_minmax", dp.SampleDefinitionWithFloat())
    for i in range(2):
        p.insert(sorted_columns(30_000, 1400 + i, t0=i * 30_000, cards=(3, 5), with_float=True), row_group_size=10_000)
    fv = lp.Col("floatvalue")
    for aggs, fcols in (([lp.Sum(val), lp.Min(val)], ()), ([lp.Max(val), lp.Count(val)], ()), ([lp.Sum(fv), lp.Sum(val)], ("sum(floatvalue)",))):
        run4(p, lambda q: q.Aggregate(aggs, KEYS), fcols)
        st = prefix_stats(p, None, aggs, KEYS)
        assert st["row_groups_prefix"] == 0 and st["row_groups_runs"] == st["row_groups"] > 0


def test_prepared_query_reexecuted_and_after_a_new_part(pair):
    p = pair("prefix_cache")
    n = 30_000
    eng, lib = p.store.engine, _lib.load()
    names = ["labels.a", "labels.b", "sum(value)", "count(value)"]

    def execute(q):
        res = C.c_void_p()
        _lib.check(lib.fgpu_query_execute(eng.handle, q, eng.table_watermark(p.name), C.byref(res)))
        st = eng.stats(res)
        out = rows_of(list(eng.drain(res)), names)
        lib.fgpu_result_free(res)
        return out, st

    p.insert(sorted_columns(n, 1500, cards=(3, 5)), row_group_size=11_000)
    q, keep = GPUScan(eng, p.name, None, _lib.PLAN_AGGREGATE, KEYS, AGGS).prepare()
    try:
        first, st = execute(q)
        again, st2 = execute(q)  # the cached Execute re-issues the launches
        got, exp = p.run(lambda b: b.Aggregate(AGGS, KEYS))
        assert first == again == rows_of(exp, names) == rows_of(got, names) and len(first) > 0
        assert st["row_groups_prefix"] == st2["row_groups_prefix"] == st["row_groups"] > 0
        assert st["rows_selected"] == st2["rows_selected"] == n
        p.insert(sorted_columns(n, 1501, t0=n, cards=(4, 7)), row_group_size=9_000)  # new part, new dictionary entries
        second, st = execute(q)
        third, _ = execute(q)
        got, exp = p.run(lambda b: b.Aggregate(AGGS, KEYS))
        assert second == third == rows_of(exp, names) and second != first
        assert st["row_groups_prefix"] == st["row_groups"] > 3
    finally:
        lib.fgpu_query_free(q)
