"""The exact Arrow layout of every result exporter: per column its type, the dictionary values in order, the raw
indices (0 under a NULL), null_count, and a validity buffer exactly when a row is NULL.

Expected values come from the generated input rows; the order of a table's dictionary comes from fgpu_dict_export.
A dictionary key column exports either the table's whole dictionary or only the values the result uses, in
dictionary (id) order: the whole one on the cached dense path when the dictionary has at most 4096 values, and on
fgpu_part_decode_column; the used values everywhere else."""
import ctypes as C

import numpy as np
import pyarrow as pa
import pytest

from frostdb_b200 import _lib
from frostdb_b200 import dynparquet as dp
from frostdb_b200 import logicalplan as lp
from frostdb_b200.physicalplan import GPUScan
from frostdb_b200.store import GPUEngine, comm_setup
from tests.test_multirank_host import union_in_rank_order
from tests.util import make_columns

pytestmark = pytest.mark.gpu

N = 20_000  # rows per part
LABELS = {"a": (6, 0.1), "b": (40, 0.0), "big": (6000, 0.05)}  # name -> (cardinality, NULL probability)
SUM, COUNT = lp.Sum(lp.Col("value")), lp.Count(lp.Col("value"))
NOTHING = lp.Col("timestamp").Lt(lp.Literal(0))


def schema():
    s = dp.SampleDefinitionWithFloat()
    s.columns.append(dp.ColumnDefinition("n64", dp.TYPE_INT64, nullable=True))
    return s


def part_columns(seed, t0):
    cols = make_columns(N, seed, LABELS, with_float=True, float_null_p=0.1, t0=t0)
    rng = np.random.default_rng(seed + 1)
    cols["n64"] = [None if rng.random() < 0.2 else int(v) for v in rng.integers(-50, 50, N)]
    return cols


def rows_of_input(parts):
    """Input rows as dicts: label values as bytes (None for NULL), the other columns as Python values."""
    out = []
    for cols in parts:
        labels = {f"labels.{n}": [None if i < 0 else cols[f"labels.{n}"][1][i].encode() for i in cols[f"labels.{n}"][0]] for n in LABELS}
        fv = cols["floatvalue"].to_pylist()
        for r in range(N):
            row = {k: v[r] for k, v in labels.items()}
            row.update(timestamp=int(cols["timestamp"][r]), value=int(cols["value"][r]), floatvalue=fv[r], n64=cols["n64"][r])
            out.append(row)
    return out


def expected_aggregate(rows, keys, where):
    groups = {}
    for r in rows:
        if where(r):
            g = groups.setdefault(tuple(r[k] for k in keys), [0, 0])
            g[0] += r["value"]
            g[1] += 1
    return [k + tuple(v) for k, v in groups.items()]


def ordered(rows):
    return sorted(rows, key=lambda r: tuple((x is None, x) for x in r))


def dict_layout(arr, dictionary):
    """Checks a dictionary key column against the dictionary it must export; returns its values per row."""
    assert arr.type == pa.dictionary(pa.uint32(), pa.binary())
    assert arr.dictionary.to_pylist() == dictionary
    assert (arr.buffers()[0] is None) == (arr.null_count == 0)
    idx = np.frombuffer(arr.buffers()[1], dtype=np.uint32, count=len(arr) + arr.offset)[arr.offset:]
    valid = arr.is_valid().to_pylist()
    assert arr.null_count == valid.count(False)
    assert all(i == 0 for i, v in zip(idx, valid) if not v), "index 0 under a NULL"
    return [dictionary[i] if v else None for i, v in zip(idx, valid)]


def value_layout(arr, typ):
    assert arr.type == typ
    assert (arr.buffers()[0] is None) == (arr.null_count == 0)
    return arr.to_pylist()


def dictionaries(eng, table, keys):
    return {k: eng.dict_export(table, k) for k in keys if k.startswith("labels.")}


def check_record(batches, names, dicts, whole, exp_rows, types=None):
    """`whole`: the key columns that export the whole dictionary (the others: the values the result uses)."""
    if not exp_rows:
        assert batches == []
        return
    assert len(batches) == 1
    b = batches[0]
    assert b.schema.names == names
    cols = []
    for i, n in enumerate(names):
        if n in dicts:
            d = dicts[n]
            used = {r[i] for r in exp_rows if r[i] is not None}
            cols.append(dict_layout(b.column(i), d if n in whole else [v for v in d if v in used]))
        else:
            cols.append(value_layout(b.column(i), (types or {}).get(n, pa.int64())))
    assert ordered(zip(*cols)) == ordered(exp_rows)


class Query:
    """One prepared query on one engine; execute() returns its drained records."""

    def __init__(self, eng, table, filt, kind, gexprs, aggs):
        self.eng, self.table = eng, table
        self.q, self.keep = GPUScan(eng, table, filt, kind, gexprs, aggs).prepare()

    def execute(self):
        lib = _lib.load()
        res = C.c_void_p()
        _lib.check(lib.fgpu_query_execute(self.eng.handle, self.q, self.eng.table_watermark(self.table), C.byref(res)))
        try:
            out = list(self.eng.drain(res))
            self.stats = self.eng.stats(res)
            return out
        finally:
            lib.fgpu_result_free(res)

    def free(self):
        _lib.load().fgpu_query_free(self.q)


@pytest.fixture()
def single():
    """A fresh engine (so that the first Execute of a plan compiles it) holding two parts of one table."""
    parts = [part_columns(11, 0), part_columns(12, N)]
    eng = GPUEngine(0)
    bufs = [dp.write_part(schema(), p, row_group_size=7_000) for p in parts]
    for b in bufs:
        eng.put_parquet("t", b)
    yield eng, rows_of_input(parts), bufs
    eng.close()


AGG_CASES = {
    # keys, filter (plan, host), the keys the cached dense path exports whole
    "small": (["labels.a", "labels.b"], (None, lambda r: True), {"labels.a", "labels.b"}),
    "big_subset": (["labels.big"], (lp.Col("timestamp").Lt(lp.Literal(N // 2)), lambda r: r["timestamp"] < N // 2), set()),
    "hash": (["labels.a", "value"], (lp.Col("timestamp").GtEq(lp.Literal(N // 3)), lambda r: r["timestamp"] >= N // 3), set()),
}


@pytest.mark.parametrize("cache", ["cached", "no_exec_cache"])
@pytest.mark.parametrize("case", sorted(AGG_CASES))
def test_aggregate_columns(single, monkeypatch, case, cache):
    eng, rows, _ = single
    if cache == "no_exec_cache":
        monkeypatch.setenv("FROSTGPU_NO_EXEC_CACHE", "1")
    keys, (filt, where), whole = AGG_CASES[case]
    if cache == "no_exec_cache" or case == "hash":
        whole = set()
    names = keys + [SUM.Name(), COUNT.Name()]
    dicts = dictionaries(eng, "t", keys)
    exp = expected_aggregate(rows, keys, where)
    assert any(None in r[:len(keys)] for r in exp), "a NULL group"
    if case == "big_subset":
        assert len({r[0] for r in exp if r[0] is not None}) < len(dicts["labels.big"]) - 100
    q = Query(eng, "t", filt, _lib.PLAN_AGGREGATE, [lp.Col(k) for k in keys], [SUM, COUNT])
    try:
        for _ in range(3):  # the first Execute compiles the plan, the later ones run it cached
            check_record(q.execute(), names, dicts, whole, exp)
    finally:
        q.free()
    empty = Query(eng, "t", NOTHING, _lib.PLAN_AGGREGATE, [lp.Col(k) for k in keys], [SUM, COUNT])
    try:
        for _ in range(2):
            assert empty.execute() == []
    finally:
        empty.free()


ROW_TYPES = {"floatvalue": pa.float64()}


@pytest.mark.parametrize("take", ["take", "no_take"])
def test_filter_columns(single, monkeypatch, take):
    eng, rows, _ = single
    if take == "no_take":
        monkeypatch.setenv("FROSTGPU_NO_TAKE", "1")
        names = ["labels.a", "labels.big", "value", "n64", "floatvalue"]  # NULLs in every column but value
    else:
        names = ["value", "timestamp"]  # the take kernels only project PLAIN int64 columns without NULLs
    lo, hi = N // 4, N + N // 3
    filt = lp.And(lp.Col("timestamp").GtEq(lp.Literal(lo)), lp.Col("timestamp").Lt(lp.Literal(hi)))
    exp = [tuple(r[n] for n in names) for r in rows if lo <= r["timestamp"] < hi]
    dicts = dictionaries(eng, "t", names)
    q = Query(eng, "t", filt, _lib.PLAN_FILTER, [lp.Col(n) for n in names], [])
    try:
        for _ in range(2):
            check_record(q.execute(), names, dicts, set(), exp, ROW_TYPES)
        launches = q.stats["kernel_launches"]
        if take == "take":  # the take kernels ran: k_rows alone is fewer launches
            monkeypatch.setenv("FROSTGPU_NO_TAKE", "1")
            check_record(q.execute(), names, dicts, set(), exp, ROW_TYPES)
            assert launches > q.stats["kernel_launches"]
            monkeypatch.delenv("FROSTGPU_NO_TAKE")
    finally:
        q.free()
    empty = Query(eng, "t", NOTHING, _lib.PLAN_FILTER, [lp.Col(n) for n in names], [])
    try:
        assert empty.execute() == []
    finally:
        empty.free()


def test_decode_columns(single):
    eng, _, bufs = single
    t = dp.read_part(bufs[1])  # (the rows in the order the part stores them)
    for col in ("labels.a", "labels.big"):
        arr = eng.decode_column("t", 1, col)
        got = dict_layout(arr, eng.dict_export("t", col))  # the whole dictionary
        assert got == [None if v is None else v.encode() for v in t.column(col).to_pylist()]
        assert arr.null_count > 0
    for col, typ in (("n64", pa.int64()), ("floatvalue", pa.float64()), ("value", pa.int64())):
        arr = eng.decode_column("t", 1, col)
        assert value_layout(arr, typ) == t.column(col).to_pylist()
        assert (arr.null_count > 0) == (col != "value")


# ---- two ranks: two contexts on one GPU ---------------------------------------------------------------------------
MR_CASES = {"dense": ["labels.a", "labels.b"], "hash": ["labels.a", "value"]}


@pytest.fixture()
def ranks():
    parts = [part_columns(21, 0), part_columns(22, N)]
    bufs = [dp.write_part(schema(), p, row_group_size=7_000) for p in parts]
    dict_cols = [f"labels.{n}" for n in LABELS]
    unions = {c: union_in_rank_order([_lib.parquet_dict_values(b, c) for b in bufs]) for c in dict_cols}
    engines = [GPUEngine(0), GPUEngine(0)]
    for e, b in zip(engines, bufs):
        for c in dict_cols:
            e.dict_preload("t", c, unions[c])
        e.put_parquet("t", b)
    yield engines, rows_of_input(parts)
    for e in engines:
        e.close()


@pytest.mark.parametrize("mode", sorted(MR_CASES))
def test_merge_partials_columns(ranks, mode):
    import torch
    lib = _lib.load()
    engines, rows = ranks
    keys = MR_CASES[mode]
    names = keys + [SUM.Name(), COUNT.Name()]
    exp = expected_aggregate(rows, keys, lambda r: True)
    qs = [Query(e, "t", None, _lib.PLAN_AGGREGATE, [lp.Col(k) for k in keys], [SUM, COUNT]) for e in engines]
    partials = []
    try:
        for q in qs:
            res, ptr, nbytes = C.c_void_p(), C.c_void_p(), C.c_uint64()
            _lib.check(lib.fgpu_query_execute_partial(q.eng.handle, q.q, q.eng.table_watermark("t"), C.byref(res), C.byref(ptr), C.byref(nbytes)))
            partials.append((res, ptr.value, nbytes.value))
        nb = partials[0][2]
        assert partials[1][2] == nb
        class DevMem:  # a partial table, as torch sees device memory it does not own
            def __init__(self, p):
                self.__cuda_array_interface__ = {"shape": (nb // 8,), "typestr": "<i8", "data": (p, False), "version": 2}
        gathered = torch.empty(2 * nb // 8, dtype=torch.int64, device="cuda")  # the tables back to back, as an all-gather leaves them
        for i, (_, ptr, _) in enumerate(partials):
            gathered[i * nb // 8:(i + 1) * nb // 8].copy_(torch.as_tensor(DevMem(ptr), device="cuda"))
        torch.cuda.synchronize()
        _lib.check(lib.fgpu_result_merge_partials(engines[0].handle, partials[0][0], gathered.data_ptr(), nb, 2))
        check_record(list(engines[0].drain(partials[0][0])), names, dictionaries(engines[0], "t", keys), set(), exp)
    finally:
        for res, _, _ in partials:
            lib.fgpu_result_free(res)
        for q in qs:
            q.free()


@pytest.mark.parametrize("mode", sorted(MR_CASES))
def test_collective_columns(ranks, mode):
    lib = _lib.load()
    engines, rows = ranks
    keys = MR_CASES[mode]
    names = keys + [SUM.Name(), COUNT.Name()]
    whole = set(keys) if mode == "dense" else set()  # dense collective plans are cached
    comm_setup(engines, slot_bytes=16 << 20)
    qs = [Query(e, "t", None, _lib.PLAN_AGGREGATE, [lp.Col(k) for k in keys], [SUM, COUNT]) for e in engines]
    try:
        for filt, where in ((None, lambda r: True), (NOTHING, lambda r: False)):
            if filt is not None:
                for q in qs:
                    q.free()
                qs = [Query(e, "t", filt, _lib.PLAN_AGGREGATE, [lp.Col(k) for k in keys], [SUM, COUNT]) for e in engines]
            exp = expected_aggregate(rows, keys, where)
            for _ in range(2):  # the first run compiles the plan, the second runs it cached
                pend = [q.eng.execute_collective_begin(q.q, q.eng.table_watermark("t")) for q in qs]
                for e, res in zip(engines, pend):
                    e.execute_collective_end(res)
                    got = list(e.drain(res))
                    lib.fgpu_result_free(res)
                    check_record(got, names, dictionaries(e, "t", keys), whole, exp)
    finally:
        for q in qs:
            q.free()
        for e in engines:
            e.comm_close()
