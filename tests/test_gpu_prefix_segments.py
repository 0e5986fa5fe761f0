"""The prefix path's segment table: a compiled plan enumerates once the segments (maximal stretches of one row group with
one dense slot) of its all-pass row groups, grouped by slot, and every Execute stores each slot's rows and Sums from
that table in place of the table initialisation.  Every case is compared with the oracle and with the prefix path
switched off (FROSTGPU_NO_PREFIX), and asserts that the prefix path took the row groups it is about."""
import ctypes as C

import numpy as np
import pytest

from frostdb_b200 import _lib
from frostdb_b200 import dynparquet as dp
from frostdb_b200 import logicalplan as lp
from frostdb_b200.physicalplan import GPUScan
from frostdb_b200.store import GPUEngine, comm_setup
from tests.oracle_scan import OracleEngine, OracleTableHandle, oracle_query
from tests.test_gpu_runs import AGGS, KEYS, pair, sorted_columns  # noqa: F401  (pair: fixture)
from tests.test_gpu_runs_narrow import EXTREMES, part_with_chunks
from tests.test_gpu_runs_prefix import prefix_stats, run4
from tests.test_multirank_host import union_in_rank_order
from tests.util import rows_of

pytestmark = pytest.mark.gpu

ts, val = lp.Col("timestamp"), lp.Col("value")
KEYS3 = KEYS + [lp.Col("labels.c")]


def check(p, filt, keys, aggs=AGGS):
    build = (lambda q: q.Filter(filt).Aggregate(aggs, keys)) if filt is not None else (lambda q: q.Aggregate(aggs, keys))
    run4(p, build)
    return prefix_stats(p, filt, aggs, keys)


def test_group_runs_across_row_groups_and_windows(pair):
    """Skewed groups: long runs cross row-group boundaries (each row group keeps its own segments) and the windows the
    build cuts (about 32 run starts each), short ones share a window."""
    p = pair("segs_windows")
    n = 300_000
    for i in range(2):
        p.insert(sorted_columns(n, 2100 + i, t0=i * n, cards=(6, 150)), row_group_size=70_001)
    for keys in ([], KEYS[:1], KEYS):
        st = check(p, None, keys)
        assert st["row_groups_prefix"] == st["row_groups"] > 8


def test_zero_to_three_keys_and_empty_slots(pair):
    """0, 1, 2 and 3 keys; the dense table has slots for every combination of dictionary ids, most without rows, next to
    slots with segments: those must come out empty, not with a stale or initial value."""
    p = pair("segs_keys")
    n = 120_000
    for i in range(2):
        p.insert(sorted_columns(n, 2200 + i, t0=i * n, cards=(5, 40), third=4, run_scale=2.0), row_group_size=40_000)
    for keys in ([], KEYS[:1], KEYS, KEYS3):
        for aggs in (AGGS, [lp.Sum(val), lp.Sum(ts)], [lp.Count(val)]):
            st = check(p, None, keys, aggs)
            assert st["row_groups_prefix"] > 0
    st = check(p, None, KEYS)
    assert 0 < st["groups"] < 6 * 41  # (5 + 1) x (40 + 1) dense slots


def test_null_keys_land_in_slot_zero(pair):
    p = pair("segs_nulls")
    n = 60_000
    for i in range(2):
        cols = sorted_columns(n, 2300 + i, t0=i * n, cards=(4, 9))
        rng = np.random.default_rng(2300 + i)
        for name, pnull in (("labels.a", 0.2), ("labels.b", 0.35)):
            idx = cols[name][0].copy()
            idx[rng.random(n) < pnull] = -1
            cols[name] = (idx, cols[name][1])
        p.insert(cols, row_group_size=25_000)
    for keys in (KEYS, KEYS[:1], [lp.Col("labels.b")]):
        st = check(p, None, keys)
        assert st["row_groups_prefix"] == st["row_groups"] > 0


def test_prefix_runs_and_tile_row_groups_in_one_plan(pair):
    """One Execute with all-pass row groups (k_runs_prefix, which initialises the table), row groups filtered row by row
    (k_runs_tma) and an unsorted part (k_tile_agg): the later launches add onto the stored slots."""
    p = pair("segs_mixed")
    n = 60_000
    # a sorted part's row groups each span its whole time range: the filter cuts into the first and the last part
    # (filtered row by row) and leaves the third all-pass; the second is in arrival order (bit-packed keys)
    p.insert(sorted_columns(n, 2400, cards=(4, 30)), row_group_size=15_000)
    p.insert(sorted_columns(n, 2401, t0=n, cards=(4, 30)), sort=False, row_group_size=15_000)
    p.insert(sorted_columns(n, 2402, t0=2 * n, cards=(4, 30)), row_group_size=15_000)
    p.insert(sorted_columns(n, 2403, t0=3 * n, cards=(4, 30)), row_group_size=15_000)
    f = lp.And(ts.GtEq(lp.Literal(7_000)), ts.Lt(lp.Literal(4 * n - 9_000)))
    st = check(p, f, KEYS)
    assert 0 < st["row_groups_prefix"] < st["row_groups_runs"]
    assert st["row_groups_tiles"] > 0
    assert st["rows_selected"] == 4 * n - 16_000
    st = check(p, f, KEYS, [lp.Sum(val)])
    assert st["row_groups_prefix"] > 0 and st["row_groups_tiles"] > 0


def test_wrapping_sums_at_the_ends_of_int64(pair):
    p = pair("segs_extremes")
    p.insert(part_with_chunks(EXTREMES, 23), row_group_size=6_000)
    for keys in (KEYS, KEYS[:1], []):
        st = check(p, None, keys, [lp.Sum(val), lp.Count(val), lp.Sum(ts)])
        assert st["row_groups_prefix"] == st["row_groups"] == len(EXTREMES)


def test_prepared_query_repeats_exactly_and_is_rebuilt_for_a_new_part(pair):
    """Five Executes of one prepared query give the same record (a missed initialisation would add the sums twice),
    and after a new part the rebuilt plan answers for both parts."""
    p = pair("segs_cache")
    n = 50_000
    eng, lib = p.store.engine, _lib.load()
    names = ["labels.a", "labels.b", "sum(value)", "count(value)"]

    def execute(q):
        res = C.c_void_p()
        _lib.check(lib.fgpu_query_execute(eng.handle, q, eng.table_watermark(p.name), C.byref(res)))
        st = eng.stats(res)
        out = rows_of(list(eng.drain(res)), names)
        lib.fgpu_result_free(res)
        return out, st

    p.insert(sorted_columns(n, 2500, cards=(3, 12)), row_group_size=12_000)
    q, keep = GPUScan(eng, p.name, None, _lib.PLAN_AGGREGATE, KEYS, AGGS).prepare()
    try:
        runs = [execute(q) for _ in range(5)]
        got, exp = p.run(lambda b: b.Aggregate(AGGS, KEYS))
        assert all(r == runs[0][0] for r, _ in runs) and runs[0][0] == rows_of(exp, names) and len(runs[0][0]) > 0
        assert all(st["rows_selected"] == n and st["row_groups_prefix"] == st["row_groups"] > 0 for _, st in runs)
        # the cached Execute has no table-init launch: the prefix launch stores every slot
        assert runs[-1][1]["kernel_launches"] < runs[0][1]["kernel_launches"]
        p.insert(sorted_columns(n, 2501, t0=n, cards=(5, 17)), row_group_size=9_000)  # new part, new dictionary entries
        again = [execute(q) for _ in range(3)]
        got, exp = p.run(lambda b: b.Aggregate(AGGS, KEYS))
        assert all(r == again[0][0] for r, _ in again) and again[0][0] == rows_of(exp, names) != runs[0][0]
        assert again[-1][1]["rows_selected"] == 2 * n and again[-1][1]["row_groups_prefix"] == again[-1][1]["row_groups"]
    finally:
        lib.fgpu_query_free(q)


def test_collective_execute_over_prefix_row_groups(built_lib):
    """Two contexts on one GPU, each with sorted parts of its own time range: every rank's partial table comes from
    the prefix launch (cached from the second Execute on), and both end with the oracle's result."""
    schema = dp.SampleDefinition()
    per = 40_000
    shards = [[dp.write_part(schema, sorted_columns(per, 2600 + 2 * r + j, t0=(2 * r + j) * per, cards=(4, 20)), row_group_size=10_000)
               for j in range(2)] for r in range(2)]
    unions = {c: union_in_rank_order([[v for b in sh for v in _lib.parquet_dict_values(b, c)] for sh in shards]) for c in ("labels.a", "labels.b")}
    engines = [GPUEngine(0) for _ in shards]
    oe = OracleEngine(threads=2)
    ot = OracleTableHandle(oe, "t", schema)
    try:
        for e, sh in zip(engines, shards):
            for c, u in unions.items():
                e.dict_preload("t", c, u)
            for b in sh:
                e.put_parquet("t", b)
                ot.InsertParquet(b)
        comm_setup(engines, slot_bytes=8 << 20)
        aggs = [lp.Sum(val), lp.Count(val)]
        names = [k.Name() for k in KEYS] + [a.Name() for a in aggs]
        for f in (None, ts.GtEq(lp.Literal(3_000))):  # (rank 0: its first part filtered row by row)
            exp = []
            oracle_query(oe, "t").Filter(f).Aggregate(aggs, KEYS).Execute(None, lambda c, r: exp.append(r))
            scans = [GPUScan(e, "t", f, _lib.PLAN_AGGREGATE, KEYS, aggs) for e in engines]
            prepared = [s.prepare() for s in scans]
            for rep in range(3):  # both halves issued separately: the ranks share one device (see test_gpu_multirank)
                pend = [engines[r].execute_collective_begin(prepared[r][0], engines[r].table_watermark("t")) for r in range(2)]
                for r in range(2):
                    engines[r].execute_collective_end(pend[r])
                    st = engines[r].stats(pend[r])
                    got = [scans[r].renamed(b) for b in engines[r].drain(pend[r])]
                    built_lib.fgpu_result_free(pend[r])
                    assert rows_of(got, names) == rows_of(exp, names), (f is not None, r, rep)
                    assert st["row_groups_prefix"] > 0
            for q, keep in prepared:
                built_lib.fgpu_query_free(q)
        for e in engines:
            e.comm_close()
    finally:
        oe.close()
        for e in engines:
            e.close()
