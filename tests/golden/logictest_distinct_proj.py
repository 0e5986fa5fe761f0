"""Golden vectors of Distinct over boolean expression keys, transcribed from the reference's end-to-end tests.

Source: logictest/testdata/exec/distinct/{distinct_proj,distinct_partial_scan_opt} (cockroach `datadriven` files run by
logictest/runner.go).  Same format as logictest_cases.py (`case` / `insert` / `exec_`), kept in a list of its own.
`select distinct(a, b, value > 0)` is Builder.Distinct(a, b, value > 0) (sqlparse/visitor.go): a Projection of the
same expressions, where a comparison is a boolean column named after it (project.go:397-467), then the Distinction.
One insert block = one InsertRecord = one part.
"""
from frostdb_b200.logicalplan import Col, Literal

DEFAULT = "default"  # dynparquet.SampleDefinitionWithFloat()

CASES = []


def case(source, schema=DEFAULT):
    c = {"source": source, "schema": schema, "steps": []}
    CASES.append(c)
    return c


def insert(c, cols, rows):
    c["steps"].append(("insert", cols, [r.split() for r in rows]))


def exec_(c, line, sql, build, expected, unordered=False, kind="distinct"):
    c["steps"].append(("exec", {"line": line, "sql": sql, "build": build, "expected": [r.split() for r in expected],
                                "unordered": unordered, "kind": kind}))


# ---------------------------------------------------------------------------------------------------
# exec/distinct/distinct_proj
# ---------------------------------------------------------------------------------------------------
_proj = case("logictest/testdata/exec/distinct/distinct_proj")
_cols = ["labels.label1", "labels.label2", "timestamp", "value"]
insert(_proj, _cols, ["value1 value2 1 0",
                      "value1 value2 2 0"])
# always true projection
exec_(_proj, 11, "select distinct(labels.label1, labels.label2, timestamp > 0)",
      lambda q: q.Distinct(Col("labels.label1"), Col("labels.label2"), Col("timestamp").Gt(Literal(0))),
      ["value1 value2 true"])
# always false projection
exec_(_proj, 17, "select distinct(labels.label1, labels.label2, value > 0)",
      lambda q: q.Distinct(Col("labels.label1"), Col("labels.label2"), Col("value").Gt(Literal(0))),
      ["value1 value2 false"])
insert(_proj, _cols, ["value2 value2 1 1",
                      "value2 value2 2 2"])
# mixed binary projection
exec_(_proj, 28, "select distinct(labels.label1, labels.label2, value > 0)",
      lambda q: q.Distinct(Col("labels.label1"), Col("labels.label2"), Col("value").Gt(Literal(0))),
      ["value1 value2 false", "value2 value2 true"], unordered=True)

# ---------------------------------------------------------------------------------------------------
# exec/distinct/distinct_partial_scan_opt: the second part's row group is one the reference's scan layer answers
# itself (every value > 0), the first is not; only the result is pinned
# ---------------------------------------------------------------------------------------------------
_partial = case("logictest/testdata/exec/distinct/distinct_partial_scan_opt")
_cols = ["labels.label1", "timestamp", "value"]
insert(_partial, _cols, ["value1 0 1",
                         "value2 1 1"])
insert(_partial, _cols, ["value2 1 1",
                         "value2 1 1"])
exec_(_partial, 22, "select distinct(labels.label1, timestamp, value > 0)",
      lambda q: q.Distinct(Col("labels.label1"), Col("timestamp"), Col("value").Gt(Literal(0))),
      ["value1 0 true", "value2 1 true"], unordered=True)
