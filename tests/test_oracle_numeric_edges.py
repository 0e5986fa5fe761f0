"""The CPU oracle (1 and 4 worker threads) against the plain reference of tests/numeric_edges.py on int64 literals at the
ends of the domain, fused ranges, int columns against float literals, IEEE specials and wrapping sums; and the engine's
statistics decision (fgpu_rowgroup_leaf_mode) at the ends of int64 against a Python statement of its rule."""
import ctypes as C
import itertools

import pytest

from frostdb_b200 import dynparquet as dp
from frostdb_b200 import logicalplan as lp
from tests import numeric_edges as ne
from tests.oracle_scan import OracleEngine, OracleTableHandle, oracle_query

N_ROWS = 2 * ne.RG * len(ne.INT_CHUNKS)


@pytest.fixture(scope="module")
def edges():
    """One sorted and one unsorted part with the same value chunks; the oracle at 1 and 4 threads."""
    parts = [ne.int_part(ne.INT_CHUNKS, 11, sort=True), ne.int_part(ne.INT_CHUNKS, 12, sort=False, t0=N_ROWS // 2, part=1)]
    bufs = [ne.write(parts[0], sort=True), ne.write(parts[1], sort=False)]
    engines = {}
    for threads in (1, 4):
        eng = OracleEngine(threads=threads)
        t = OracleTableHandle(eng, "edges", dp.SampleDefinitionWithFloat())
        for b in bufs:
            t.InsertParquet(b)
        engines[threads] = eng
    yield engines, [ne.physical(p) for p in parts]
    for eng in engines.values():
        eng.close()


def oracle_agg(eng, filt, keys, aggs, table="edges"):
    out = []
    q = oracle_query(eng, table)
    if filt is not None:
        q = q.Filter(filt)
    q.Aggregate(aggs, [lp.Col(k) for k in keys]).Execute(None, lambda c, r: out.append(r))
    return ne.result_map(out, keys, aggs)


def check(engines, phys, filters, aggs, threads, keys=ne.KEYS):
    for f in filters:
        if threads == 4 and ne.has_nan_minmax(aggs):
            continue
        exp = ne.reference(phys, f, keys, aggs)
        got = oracle_agg(engines[threads], f, keys, aggs)
        ne.assert_same_result(got, exp, aggs, f"threads={threads} filter {f.Name() if f is not None else None}")


@pytest.mark.parametrize("threads", [1, 4])
def test_int64_literal_edges(edges, threads):
    engines, phys = edges
    check(engines, phys, ne.int_edge_filters(N_ROWS), ne.AGG_INT, threads)


@pytest.mark.parametrize("threads", [1, 4])
def test_fused_conjunctions(edges, threads):
    engines, phys = edges
    check(engines, phys, ne.fused_filters(), ne.AGG_INT, threads)


@pytest.mark.parametrize("threads", [1, 4])
def test_int_column_against_float_literals(edges, threads):
    engines, phys = edges
    check(engines, phys, ne.int_float_filters(), ne.AGG_INT, threads)


@pytest.mark.parametrize("threads", [1, 4])
def test_float_specials(edges, threads):
    engines, phys = edges
    check(engines, phys, [None] + ne.float_filters(), ne.AGG_FLOAT, threads)
    check(engines, phys, [None] + ne.float_filters(), ne.AGG_FLOAT_SUM + [lp.Min(lp.Col(ne.V))], threads)
    # the dataset holds what the cases are about
    exp = ne.reference(phys, None, ne.KEYS, ne.AGG_FLOAT)
    sums = [v[0] for v in exp.values()]
    assert any(s != s for s in sums) and ne.INF in sums and any(0 < abs(s) < 1e-300 for s in sums)
    assert -ne.INF in [v[1] for v in exp.values()] and ne.DBL_MAX in [v[2] for v in exp.values()]


def test_filter_only_rows_in_order(edges):
    engines, phys = edges
    names = [ne.T, ne.V, ne.F]
    for f in ne.fused_filters() + [ne.leaf(ne.V, op, x) for op in ne.OPS for x in ne.EDGE_LITERALS]:
        out = []
        oracle_query(engines[1], "edges").Filter(f).Project(*[lp.Col(n) for n in names]).Execute(None, lambda c, r: out.append(r))
        ne.assert_same_rows(ne.record_rows(out, names), ne.reference_rows(phys, f, names), f.Name())


@pytest.mark.parametrize("threads", [1, 4])
def test_wrapping_sums(threads):
    eng = OracleEngine(threads=threads)
    try:
        t = OracleTableHandle(eng, "wrap", dp.SampleDefinition())
        parts = [ne.wrap_part(20_000, 5), ne.wrap_part(20_000, 6, t0=20_000, ka=300, kb=200, used=(5, 7))]
        for p in parts:
            t.InsertParquet(dp.write_part(dp.SampleDefinition(), p, sort=False, row_group_size=7_000))
        phys = [ne.physical(p) for p in parts]
        aggs = ne.AGG_INT
        for p in phys:  # running sums leave int64 many times
            assert max(abs(s) for s in itertools.accumulate(p["value"][:1000].tolist())) > 4 * ne.I64_MAX
        for f in (None, ne.leaf(ne.T, lp.OpLt, 30_000), lp.Or(ne.leaf(ne.V, lp.OpLt, 0), ne.leaf(ne.T, lp.OpGt, 35_000))):
            exp = ne.reference(phys, f, ne.KEYS, aggs)
            ne.assert_same_result(oracle_agg(eng, f, ne.KEYS, aggs, "wrap"), exp, aggs, f"wrap {f.Name() if f is not None else None}")
    finally:
        eng.close()


def _rule(op, lit, mn, mx):
    """What statistics may decide for `x op lit` on a chunk with non-null values in [mn, mx]: NONE (2) only if no value
    in [mn, mx] matches; ALL (1) only if every value in [mn, mx] matches and there are no NULLs."""
    match = {lp.OpEq: lambda x: x == lit, lp.OpNotEq: lambda x: x != lit, lp.OpLt: lambda x: x < lit,
             lp.OpLtEq: lambda x: x <= lit, lp.OpGt: lambda x: x > lit, lp.OpGtEq: lambda x: x >= lit}[op]
    # a predicate of this kind matches an interval's values either nowhere, everywhere, or somewhere: decide from the
    # ends and the literal's neighbours inside [mn, mx]
    probes = {mn, mx} | {x for x in (lit - 1, lit, lit + 1) if mn <= x <= mx}
    return {match(x) for x in probes}


def test_leaf_mode_at_the_ends_of_int64(built_lib):
    """Never drop a row group that holds a matching value; LM_ALL only if every value matches and there are no NULLs."""
    I64_MIN, I64_MAX = ne.I64_MIN, ne.I64_MAX
    ends = [I64_MIN, I64_MIN + 1, I64_MIN + 2, -2, -1, 0, 1, I64_MAX - 2, I64_MAX - 1, I64_MAX]
    bounds = [(a, b) for a in ends for b in ends if a <= b]
    seen = {0: 0, 1: 0, 2: 0}
    for op in ne.OPS:
        for lit in ne.EDGE_LITERALS:
            for mn, mx in bounds:
                for nulls in (0, 3):
                    mode = C.c_int32(-1)
                    assert built_lib.fgpu_rowgroup_leaf_mode(op, lit, 1, mn, mx, nulls, 10, C.byref(mode)) == 0
                    res = _rule(op, lit, mn, mx)
                    what = (op, lit, mn, mx, nulls, mode.value)
                    if mode.value == 2:
                        assert res == {False}, what
                    elif mode.value == 1:
                        assert res == {True} and nulls == 0, what
                    else:
                        assert mode.value == 0, what
                    seen[mode.value] += 1
    assert min(seen.values()) > 100
