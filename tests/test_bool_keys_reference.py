"""The plain reference of Distinct over boolean expression keys (tests/bool_keys_reference.py) against the reference's
own golden vectors, so that the GPU tests compare against rules the goldens confirm."""
import pyarrow as pa

from frostdb_b200 import dynparquet as dp
from frostdb_b200 import logicalplan as lp
from tests import bool_keys_reference as ref
from tests import golden_runner as gr
from tests.golden.logictest_distinct_proj import CASES


class _Recorder:
    """Builder stand-in that records the Distinct expressions an exec builds."""

    def __init__(self):
        self.exprs = None

    def Distinct(self, *exprs):
        self.exprs = list(exprs)
        return self


def _fmt(v):
    if isinstance(v, bool):
        return "true" if v else "false"
    return "null" if v is None else str(v)


def test_reference_reproduces_goldens():
    ran = 0
    for case in CASES:
        schema = gr.SCHEMAS[case["schema"]]()
        parts = []
        for step in case["steps"]:
            if step[0] == "insert":
                _, names, rows = step
                cols = gr.columns_of_insert(schema, names, rows)
                parts.append(ref.read_part(dp.write_part(schema, cols)))
                continue
            ex = step[1]
            rec = _Recorder()
            ex["build"](rec)
            got = [[_fmt(v) for v in r] for r in ref.distinct_rows(parts, rec.exprs)]
            gr.check(ex, got, ex["expected"])
            ran += 1
    assert ran == 4


def test_missing_column_rules():
    part = {"value": [1, None]}
    L = lp.Literal
    c = lp.Col("labels.nosuch")
    assert ref.eval_bool(c.Gt(L(0)), part, 0) is False
    assert ref.eval_bool(c.Eq(L(5)), part, 0) is True
    assert ref.eval_bool(c.Eq(L("x")), part, 0) is False
    assert ref.eval_bool(c.Eq(L("")), part, 0) is True
    assert ref.eval_bool(c.NotEq(L(None)), part, 0) is False
    assert ref.eval_bool(c.RegexMatch("^$"), part, 0) is True
    assert ref.eval_bool(c.RegexMatch("a"), part, 0) is False
    assert ref.eval_bool(c.Contains("a"), part, 0) is True
    assert ref.eval_bool(lp.Col("value").NotEq(L(3)), part, 1) is False  # NULL numeric: never selected
    assert ref.eval_bool(lp.Col("value").NotEq(L(float("nan"))), part, 0) is True
