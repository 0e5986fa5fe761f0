"""The host's post-aggregate projection (Projection.Callback / _eval_post) on hand-built result records against the
plain reference of tests/numeric_edges.py: int64 arithmetic that wraps, division that truncates toward zero at the
ends of int64 (INT64_MIN / 2, INT64_MIN / -1), zero divisors that give NULL, and float64 specials."""
import numpy as np
import pyarrow as pa

from frostdb_b200 import logicalplan as lp
from frostdb_b200.physicalplan import PhysicalPlan, Projection
from tests import numeric_edges as ne

I64 = [ne.I64_MIN, ne.I64_MIN + 1, -7, -2, -1, 0, 1, 2, 7, ne.I64_MAX - 1, ne.I64_MAX]
F64 = [-ne.INF, -ne.DBL_MAX, -2.5, -0.0, 0.0, ne.DENORM_MIN, 1.0, ne.DBL_MAX, ne.INF, ne.NAN, 3.0]


class _Collect(PhysicalPlan):
    def __init__(self):
        self.out = []

    def Callback(self, ctx, r):
        self.out.append(r)


def project(batch, exprs):
    p = Projection(exprs)
    c = _Collect()
    p.SetNext(c)
    p.Callback(None, batch)
    assert len(c.out) == 1
    return c.out[0]


def record():
    """Every pair of the edge values: min(value) x max(value), and two float columns."""
    a, b = zip(*[(x, y) for x in I64 for y in I64])
    fa, fb = zip(*[(x, y) for x in F64 for y in F64])
    n = len(a)
    fa, fb = (list(fa) * (n // len(fa) + 1))[:n], (list(fb) * (n // len(fb) + 1))[:n]
    return {"min(value)": np.array(a, np.int64), "max(value)": np.array(b, np.int64),
            "min(floatvalue)": np.array(fa, np.float64), "max(floatvalue)": np.array(fb, np.float64)}


def check(exprs):
    cols = record()
    names = list(cols)
    batch = pa.RecordBatch.from_arrays([pa.array(cols[n]) for n in names], names=names)
    got = project(batch, exprs)
    res = {i: tuple(cols[n][i].item() for n in names) for i in range(len(cols["min(value)"]))}
    exp = ne.post_project(res, names, exprs)
    for j, e in enumerate(exprs):
        g = got.column(j).to_pylist()
        assert got.schema.names[j] == e.Name()
        for i in range(len(g)):
            ev = exp[i][j]
            ok = (g[i] is None and ev is None) or (g[i] is not None and ev is not None and ne.same_value(g[i], ev, 0))
            assert ok, f"{e.Name()} over {res[i]}: got {g[i]!r}, expected {ev!r}"


def test_int64_division_truncates_at_the_ends_of_int64():
    mn, mx = lp.Col("min(value)"), lp.Col("max(value)")
    check([lp.Div(mn, lp.Literal(2)), lp.Div(mn, lp.Literal(-1)), lp.Div(mn, lp.Literal(-2)), lp.Div(mn, mx),
           lp.Div(mx, mn), lp.Div(mn, lp.Literal(0)), lp.Div(lp.Literal(7), mx)])


def test_int64_min_over_two_is_minus_two_to_the_62():
    batch = pa.RecordBatch.from_arrays([pa.array([ne.I64_MIN, ne.I64_MIN + 1, -3], pa.int64())], names=["min(value)"])
    got = project(batch, [lp.Div(lp.Col("min(value)"), lp.Literal(2))]).column(0).to_pylist()
    assert got == [-(1 << 62), -(1 << 62) + 1, -1]


def test_int64_add_sub_mul_wrap():
    mn, mx = lp.Col("min(value)"), lp.Col("max(value)")
    check([lp.Add(mn, mx), lp.Sub(mn, mx), lp.Mul(mn, mx), lp.Sub(lp.Literal(ne.I64_MIN), mx), lp.Mul(mx, lp.Literal(2))])


def test_float64_arithmetic_and_zero_divisors():
    fa, fb = lp.Col("min(floatvalue)"), lp.Col("max(floatvalue)")
    check([lp.Add(fa, fb), lp.Sub(fa, fb), lp.Mul(fa, fb), lp.Div(fa, fb), lp.Div(fa, lp.Literal(0.0)),
           lp.Div(fa, lp.Literal(-0.0)), lp.Div(lp.Literal(1.0), fb)])
