"""The plain Unique reference (tests/unique_reference.py) on the reference's golden, on hand cases and against pyarrow's
grouped min / max / null count, and the Unique aggregate's encoding in a plan."""
import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

from frostdb_b200 import _lib
from frostdb_b200 import logicalplan as lp
from frostdb_b200.physicalplan import GPUScan
from tests import unique_reference as ref
from tests.golden import unique_aggregation as golden

I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1


def _col(name):
    return lambda part, i: part[name][i]


def test_golden():
    got = ref.rows([golden.ROWS], [_col(c) for c in golden.GROUP_BY], [golden.AGGREGATE[1]])
    exp = sorted(zip(*(golden.EXPECTED[c] for c in golden.GROUP_BY + ["unique(example)"])))
    assert got == exp == [(1, None), (3, 3)]


@pytest.mark.parametrize("values,expected", [
    ([None], None), ([None, None], None), ([5, None, 5], None), ([None, 5], None), ([5, 5, 5], 5), ([5], 5), ([0], 0),
    ([5, 6], None), ([I64_MIN], I64_MIN), ([I64_MIN, I64_MIN], I64_MIN), ([I64_MAX, I64_MAX], I64_MAX),
    ([I64_MIN, None], None), ([I64_MAX, None], None), ([I64_MIN, I64_MAX], None), ([0, None], None),
])
def test_hand_cases(values, expected):
    assert ref.unique(values) == expected
    assert ref.grouped([("g",)] * len(values), values) == {("g",): expected}


def test_partials_give_the_same_answer_whatever_the_split():
    values = [3, 3, None, 3]
    whole = ref.unique(values)
    for cut in range(1, len(values)):
        parts = [ref.unique(values[:cut]), ref.unique(values[cut:])]
        assert ref.unique(parts) == whole is None
    assert ref.unique([ref.unique([7, 7]), ref.unique([7])]) == 7


@pytest.mark.parametrize("seed", range(6))
def test_against_pyarrow_grouped_min_max_null_count(seed):
    rng = np.random.default_rng(seed)
    n = 4000
    g = rng.integers(0, 50, n)
    pool = np.array([I64_MIN, I64_MIN + 1, -1, 0, 1, I64_MAX - 1, I64_MAX], dtype=np.int64)
    base = pool[rng.integers(0, len(pool), 50)]
    v = base[g].copy()
    flip = rng.random(n) < (0.002 if seed % 2 else 0.02)  # a few groups get a second value
    v[flip] = pool[rng.integers(0, len(pool), int(flip.sum()))]
    nulls = rng.random(n) < (0.001 if seed < 3 else 0.0)
    nulls[g == 7] |= seed == 5  # one all-NULL group
    t = pa.table({"g": g, "v": pa.array(v, mask=nulls)})
    agg = t.group_by("g").aggregate([("v", "min"), ("v", "max"), ("v", "count", pc.CountOptions(mode="only_null"))])
    exp = {}
    for k, lo, hi, nn in zip(*(agg.column(c).to_pylist() for c in ("g", "v_min", "v_max", "v_count"))):
        exp[(k,)] = lo if nn == 0 and lo == hi else None
    vals = [None if m else int(x) for x, m in zip(v, nulls)]
    assert ref.grouped([(int(k),) for k in g], vals) == exp
    assert any(x is None for x in exp.values()) and any(x is not None for x in exp.values())


def test_unique_encodes_as_agg_unique():
    assert lp.AggFuncUnique == _lib.AGG_UNIQUE
    u = lp.Unique(lp.Col("example"))
    assert u.Name() == "unique(example)"
    plan, _keep = GPUScan(None, "t", None, _lib.PLAN_AGGREGATE, [lp.Col("timestamp")], [u, lp.Sum(lp.Col("value"))])._plan()
    assert plan.n_aggs == 2
    assert [plan.aggs[i].func for i in range(2)] == [_lib.AGG_UNIQUE, _lib.AGG_SUM]
    assert plan.exprs[plan.aggs[0].expr].name == b"example"


def test_builder_passes_unique_through_and_rewrites_only_avg():
    b = lp.Builder().Scan(None, "t")
    plain = b.Aggregate([lp.Unique(lp.Col("v"))], [lp.Col("g")]).Build()
    assert [a.Func for a in plain.Aggregation.AggExprs] == [lp.AggFuncUnique]
    mixed = b.Aggregate([lp.Unique(lp.Col("v")), lp.Avg(lp.Col("v"))], [lp.Col("g")]).Build()
    assert [a.Func for a in mixed.Input.Aggregation.AggExprs] == [lp.AggFuncUnique, lp.AggFuncSum, lp.AggFuncCount]
    assert [e.Name() for e in mixed.Projection.Exprs] == ["g", "unique(v)", "avg(v)"]
