"""The N > 1 data path on one GPU: two engines (two fgpu_ctx, as two ranks would have) each own half of the
parts, preload the same dictionary union, scan into partial tables, the tables are laid out back to back
the way an all-gather leaves them, and one engine merges.  Must equal the single-engine result and the
oracle."""
import ctypes as C

import pytest

from frostdb_b200 import _lib
from frostdb_b200 import dynparquet as dp
from frostdb_b200 import logicalplan as lp
from frostdb_b200.physicalplan import GPUScan
from frostdb_b200.store import GPUEngine
from tests.oracle_scan import OracleEngine, OracleTableHandle, oracle_query
from tests.test_multirank_host import union_in_rank_order
from tests.util import make_columns, rows_of

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("groups", [["labels.a", "labels.b"], ["labels.a", "labels.big", "labels.b"]])
def test_partial_tables_merge_like_the_final_aggregate(built_lib, groups):
    import torch
    lib = built_lib
    schema = dp.SampleDefinition()
    bufs = []
    for r in range(4):  # ranks see different label windows -> different local dictionaries
        cols = make_columns(30_000, 70 + r, {"a": (5 + 3 * (r % 2), 0.1), "b": (40, 0.0), "big": (20000 + 500 * r, 0.02)}, t0=r * 30_000)
        bufs.append(dp.write_part(schema, cols, row_group_size=12_000))
    shards = [bufs[0::2], bufs[1::2]]
    key_cols = groups
    unions = {c: union_in_rank_order([[v for b in sh for v in _lib.parquet_dict_values(b, c)] for sh in shards]) for c in key_cols}
    engines = [GPUEngine(0), GPUEngine(0)]
    oe = OracleEngine(threads=2)
    try:
        ot = OracleTableHandle(oe, "t", schema)
        for e, sh in zip(engines, shards):
            for c in key_cols:
                e.dict_preload("t", c, unions[c])
            for b in sh:
                e.put_parquet("t", b)
        for b in bufs:
            ot.InsertParquet(b)
        aggs = [lp.Sum(lp.Col("value")), lp.Count(lp.Col("value")), lp.Min(lp.Col("timestamp")), lp.Max(lp.Col("value"))]
        gexprs = [lp.Col(c) for c in key_cols]
        f = lp.Col("timestamp").GtEq(lp.Literal(10_000))
        partials = []
        for e in engines:
            scan = GPUScan(e, "t", f, _lib.PLAN_AGGREGATE, gexprs, aggs)
            q, keep = scan.prepare()
            res, ptr, nbytes = C.c_void_p(), C.c_void_p(), C.c_uint64()
            _lib.check(lib.fgpu_query_execute_partial(e.handle, q, e.table_watermark("t"), C.byref(res), C.byref(ptr), C.byref(nbytes)))
            partials.append((e, q, keep, res, ptr.value, nbytes.value))
        assert partials[0][5] == partials[1][5], "partial tables must have the same layout on every rank"
        n8 = partials[0][5] // 8

        class DevMem:
            def __init__(self, p, n):
                self.__cuda_array_interface__ = {"shape": (n // 8,), "typestr": "<i8", "data": (p, False), "version": 2}
        gathered = torch.empty(2 * n8, dtype=torch.int64, device="cuda")
        for i, (_, _, _, _, ptr, nb) in enumerate(partials):
            gathered[i * n8:(i + 1) * n8].copy_(torch.as_tensor(DevMem(ptr, nb), device="cuda"))
        torch.cuda.synchronize()
        e0, q0, _, res0, _, nb = partials[0]
        _lib.check(lib.fgpu_result_merge_partials(e0.handle, res0, gathered.data_ptr(), nb, 2))
        got = list(e0.drain(res0))
        exp = []
        oracle_query(oe, "t").Filter(f).Aggregate(aggs, gexprs).Execute(None, lambda c, r: exp.append(r))
        names = key_cols + [a.Name() for a in aggs]
        assert rows_of(got, names) == rows_of(exp, names)
        for e, q, _, res, _, _ in partials:
            lib.fgpu_result_free(res)
            lib.fgpu_query_free(q)
    finally:
        oe.close()
        for e in engines:
            e.close()


def test_additive_partial_tables_reduce_in_place(built_lib):
    """Dense table of counts and integer sums: adding the ranks' tables element-wise (what an NCCL all-reduce
    does) and finalising without a gather equals the oracle; Min/Max or float sums must say "not additive"."""
    import torch
    lib = built_lib
    schema = dp.SampleDefinition()
    bufs = [dp.write_part(schema, make_columns(25_000, 80 + r, {"a": (6, 0.1), "b": (30, 0.0)}, t0=r * 25_000), row_group_size=9_000)
            for r in range(4)]
    shards = [bufs[0::2], bufs[1::2]]
    key_cols = ["labels.a", "labels.b"]
    unions = {c: union_in_rank_order([[v for b in sh for v in _lib.parquet_dict_values(b, c)] for sh in shards]) for c in key_cols}
    engines = [GPUEngine(0), GPUEngine(0)]
    oe = OracleEngine(threads=2)
    try:
        ot = OracleTableHandle(oe, "t", schema)
        for e, sh in zip(engines, shards):
            for c in key_cols:
                e.dict_preload("t", c, unions[c])
            for b in sh:
                e.put_parquet("t", b)
        for b in bufs:
            ot.InsertParquet(b)
        gexprs = [lp.Col(c) for c in key_cols]
        f = lp.Col("timestamp").Lt(lp.Literal(80_000))

        class DevMem:
            def __init__(self, p, n):
                self.__cuda_array_interface__ = {"shape": (n // 8,), "typestr": "<i8", "data": (p, False), "version": 2}

        def partials(aggs):
            out = []
            for e in engines:
                q, keep = GPUScan(e, "t", f, _lib.PLAN_AGGREGATE, gexprs, aggs).prepare()
                res, ptr, nbytes = C.c_void_p(), C.c_void_p(), C.c_uint64()
                _lib.check(lib.fgpu_query_execute_partial(e.handle, q, e.table_watermark("t"), C.byref(res), C.byref(ptr), C.byref(nbytes)))
                add = C.c_int32(-1)
                _lib.check(lib.fgpu_result_partial_is_additive(res, C.byref(add)))
                out.append((e, q, keep, res, ptr.value, nbytes.value, add.value))
            return out

        aggs = [lp.Sum(lp.Col("value")), lp.Count(lp.Col("value")), lp.Sum(lp.Col("timestamp"))]
        ps = partials(aggs)
        assert [p[6] for p in ps] == [1, 1] and ps[0][5] == ps[1][5]
        t0 = torch.as_tensor(DevMem(ps[0][4], ps[0][5]), device="cuda")
        t0 += torch.as_tensor(DevMem(ps[1][4], ps[1][5]), device="cuda")   # the all-reduce, with two "ranks" on one GPU
        torch.cuda.synchronize()
        _lib.check(lib.fgpu_result_merge_partials(ps[0][0].handle, ps[0][3], None, 0, 0))
        got = list(ps[0][0].drain(ps[0][3]))
        exp = []
        oracle_query(oe, "t").Filter(f).Aggregate(aggs, gexprs).Execute(None, lambda c, r: exp.append(r))
        names = key_cols + [a.Name() for a in aggs]
        assert rows_of(got, names) == rows_of(exp, names)
        for p in ps:
            lib.fgpu_result_free(p[3])
            lib.fgpu_query_free(p[1])
        ps = partials([lp.Sum(lp.Col("value")), lp.Max(lp.Col("value"))])
        assert [p[6] for p in ps] == [0, 0]
        for p in ps:
            lib.fgpu_result_free(p[3])
            lib.fgpu_query_free(p[1])
    finally:
        oe.close()
        for e in engines:
            e.close()


def _ranks(parts_per_rank, key_cols, per=30_000, seed=170):
    """Parts of `per` rows, contiguous time ranges per rank (rank r holds parts_per_rank[r] of them); every rank
    preloads the union of the dictionaries of `key_cols`.  Returns (engines, oracle engine, schema, per)."""
    schema = dp.SampleDefinition()
    shards, i = [], 0
    for r, n in enumerate(parts_per_rank):
        sh = []
        for _ in range(n):
            cols = make_columns(per, seed + i, {"a": (5 + 3 * (r % 2), 0.1), "b": (40, 0.0), "big": (20000 + 500 * (r % 2), 0.02)}, t0=i * per)
            sh.append(dp.write_part(schema, cols, row_group_size=12_000))
            i += 1
        shards.append(sh)
    dict_cols = [c for c in key_cols if c.startswith("labels.")]
    unions = {c: union_in_rank_order([[v for b in sh for v in _lib.parquet_dict_values(b, c)] for sh in shards]) for c in dict_cols}
    engines = [GPUEngine(0) for _ in shards]
    oe = OracleEngine(threads=2)
    ot = OracleTableHandle(oe, "t", schema)
    for e, sh in zip(engines, shards):
        for c in dict_cols:
            e.dict_preload("t", c, unions[c])
        for b in sh:
            e.put_parquet("t", b)
            ot.InsertParquet(b)
    return engines, oe


def _collective(lib, engines, oe, gexprs, aggs, filters):
    """Every rank runs the collective Execute (three times: compiled plan, then cached plan with alternating mailbox
    sets) and must end with the result of the union of all parts (= the oracle)."""
    from frostdb_b200.store import comm_setup
    comm_setup(engines, slot_bytes=48 << 20)
    n_ranks = len(engines)
    names = [g.Name() for g in gexprs] + [a.Name() for a in aggs]
    for f in filters:
        exp = []
        oracle_query(oe, "t").Filter(f).Aggregate(aggs, gexprs).Execute(None, lambda c, r: exp.append(r))
        scans = [GPUScan(e, "t", f, _lib.PLAN_AGGREGATE, gexprs, aggs) for e in engines]
        prepared = [s.prepare() for s in scans]
        # The ranks of this test share ONE device, where a rank's flag wait would keep its peers' kernels from
        # running: the two halves of the collective are issued separately, every push before the first wait.  (One
        # GPU per rank runs the fused fgpu_query_execute_collective; bench.py --gpus N does.)
        for rep in range(3):  # first run: plan compiled; later runs: cached plan, alternating mailbox sets
            pend = [engines[r].execute_collective_begin(prepared[r][0], engines[r].table_watermark("t")) for r in range(n_ranks)]
            for r in range(n_ranks):
                engines[r].execute_collective_end(pend[r])
                got = [scans[r].renamed(b) for b in engines[r].drain(pend[r])]
                lib.fgpu_result_free(pend[r])
                assert rows_of(got, names) == rows_of(exp, names), (f.Name() if f is not None else None, r, rep)
        for q, keep in prepared:
            lib.fgpu_query_free(q)
    for e in engines:
        e.comm_close()


AGGS = [lp.Sum(lp.Col("value")), lp.Count(lp.Col("value")), lp.Min(lp.Col("timestamp")), lp.Max(lp.Col("value"))]


@pytest.mark.parametrize("n_ranks,key_cols", [(2, ["labels.a", "labels.b"]), (3, ["labels.a", "labels.b"]), (2, ["labels.a", "labels.big", "labels.b"])])
def test_collective_execute_exchanges_inside_the_library(built_lib, n_ranks, key_cols):
    """The exchange inside the library: scan -> push into every rank's mailbox -> wait -> merge, per rank, no host
    collective.  Ranks are contexts on one GPU; every rank must end with the result of the union of all parts
    (= the oracle), also when the filter leaves a rank nothing to scan (in hash mode its table is then smaller than
    its peers'), and when the same prepared query runs again (cached plan, alternating mailbox sets)."""
    engines, oe = _ranks([2] * n_ranks, key_cols)
    try:
        per = 30_000
        filters = [None, lp.Col("timestamp").GtEq(lp.Literal(10_000)), lp.Col("timestamp").GtEq(lp.Literal(2 * per + 5))]
        _collective(built_lib, engines, oe, [lp.Col(c) for c in key_cols], AGGS, filters)
    finally:
        oe.close()
        for e in engines:
            e.close()


def _bucket():
    return lp.Mul(lp.Div(lp.Col("timestamp"), lp.Literal(1000)), lp.Literal(1000)).Alias("bucket")


@pytest.mark.parametrize("keys", ["big", "int64", "computed"])
def test_collective_hash_mode_on_ranks_of_unequal_size(built_lib, keys):
    """Hash-mode partial tables are sized from each rank's own visible rows: ranks of 2 and 3 parts push tables of
    different sizes, and the merge table must hold the groups of both."""
    gexprs = {"big": [lp.Col("labels.a"), lp.Col("labels.big"), lp.Col("labels.b")],
              "int64": [lp.Col("value"), lp.Col("labels.a")],
              "computed": [lp.Col("labels.a"), _bucket()]}[keys]
    engines, oe = _ranks([2, 3], [g.Name() for g in gexprs if isinstance(g, lp.Column)])
    try:
        _collective(built_lib, engines, oe, gexprs, AGGS, [None, lp.Col("timestamp").GtEq(lp.Literal(10_000))])
    finally:
        oe.close()
        for e in engines:
            e.close()


def test_three_ranks_of_distinct_int64_keys(built_lib):
    """Three ranks of 60 000 rows grouped by `timestamp`, whose every value is distinct: 180 000 groups, more than
    one rank's 131 072-slot table holds.  Collective, and through fgpu_query_execute_partial +
    fgpu_result_merge_partials(n = 3)."""
    import torch
    lib = built_lib
    engines, oe = _ranks([2, 2, 2], [])
    try:
        gexprs = [lp.Col("timestamp")]
        aggs = [lp.Sum(lp.Col("value")), lp.Count(lp.Col("value"))]
        _collective(lib, engines, oe, gexprs, aggs, [None])
        partials = []
        for e in engines:
            q, keep = GPUScan(e, "t", None, _lib.PLAN_AGGREGATE, gexprs, aggs).prepare()
            res, ptr, nbytes = C.c_void_p(), C.c_void_p(), C.c_uint64()
            _lib.check(lib.fgpu_query_execute_partial(e.handle, q, e.table_watermark("t"), C.byref(res), C.byref(ptr), C.byref(nbytes)))
            partials.append((e, q, keep, res, ptr.value, nbytes.value))
        nb = partials[0][5]
        assert all(p[5] == nb for p in partials)
        n8 = nb // 8

        class DevMem:
            def __init__(self, p, n):
                self.__cuda_array_interface__ = {"shape": (n // 8,), "typestr": "<i8", "data": (p, False), "version": 2}
        gathered = torch.empty(3 * n8, dtype=torch.int64, device="cuda")
        for i, p in enumerate(partials):
            gathered[i * n8:(i + 1) * n8].copy_(torch.as_tensor(DevMem(p[4], nb), device="cuda"))
        torch.cuda.synchronize()
        e0, _, _, res0, _, _ = partials[0]
        _lib.check(lib.fgpu_result_merge_partials(e0.handle, res0, gathered.data_ptr(), nb, 3))
        got = list(e0.drain(res0))
        exp = []
        oracle_query(oe, "t").Aggregate(aggs, gexprs).Execute(None, lambda c, r: exp.append(r))
        names = ["timestamp"] + [a.Name() for a in aggs]
        assert len(rows_of(exp, names)) == 180_000
        assert rows_of(got, names) == rows_of(exp, names)
        for _, q, _, res, _, _ in partials:
            lib.fgpu_result_free(res)
            lib.fgpu_query_free(q)
    finally:
        oe.close()
        for e in engines:
            e.close()
