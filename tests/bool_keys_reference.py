"""A plain reference for Distinct over boolean expression keys: pyarrow reads the parts, Python evaluates every row.

It restates the reference's rules without any engine or oracle code: a boolean key is the filter's bitmap for the row
(boolExprProjection, physicalplan/project.go:397-467; binaryscalarexpr.go:41-311), never NULL.
- A NULL numeric value is never selected; a comparison with a NULL literal on a numeric column selects nothing.
- A string column: `== NULL` / `!= NULL` select the NULL / non-NULL rows; any other leaf is false on a NULL row.
- A column absent from a part (SURVEY.md Appendix B.1): `== "x"` (non-empty string) false, `!= NULL` false, orderings
  false, regex as its match of "", everything else true.
"""
from __future__ import annotations

import io
import math
import re
from typing import Dict, List

import pyarrow as pa
import pyarrow.parquet as pq

from frostdb_b200 import logicalplan as lp


def read_part(buf: bytes) -> Dict[str, list]:
    t = pq.read_table(io.BytesIO(buf))
    out = {}
    for name in t.column_names:
        a = t.column(name).combine_chunks()
        if pa.types.is_dictionary(a.type):
            a = a.dictionary_decode()
        out[name] = [v.decode() if isinstance(v, bytes) else v for v in a.to_pylist()]
    return out


def _missing(e: lp.BinaryExpr) -> bool:
    v = e.Right.Value
    if e.Op == lp.OpEq:
        return not (isinstance(v, (str, bytes)) and len(v) > 0)
    if e.Op == lp.OpNotEq:
        return v is not None
    if e.Op in (lp.OpLt, lp.OpLtEq, lp.OpGt, lp.OpGtEq):
        return False
    if e.Op in (lp.OpRegexMatch, lp.OpRegexNotMatch):
        m = re.search(v, "") is not None
        return m if e.Op == lp.OpRegexMatch else not m
    return True


def _cmp(op, x, y) -> bool:
    return {lp.OpEq: x == y, lp.OpNotEq: x != y, lp.OpLt: x < y, lp.OpLtEq: x <= y, lp.OpGt: x > y, lp.OpGtEq: x >= y}[op]


def eval_bool(e: lp.Expr, part: Dict[str, list], i: int) -> bool:
    """Value of boolean expression e on row i of a part (column name -> values)."""
    if e.Op == lp.OpAnd:
        return eval_bool(e.Left, part, i) and eval_bool(e.Right, part, i)
    if e.Op == lp.OpOr:
        return eval_bool(e.Left, part, i) or eval_bool(e.Right, part, i)
    col = e.Left.ColumnName
    if col not in part:
        return _missing(e)
    x = part[col][i]
    lit = e.Right.Value
    if isinstance(x, str) or (x is None and col.startswith("labels.")) or col in ("example_type", "stacktrace"):
        if e.Op == lp.OpEq and lit is None:
            return x is None
        if e.Op == lp.OpNotEq and lit is None:
            return x is not None
        if x is None:
            return False
        if e.Op == lp.OpEq:
            return x == lit
        if e.Op == lp.OpNotEq:
            return x != lit
        if e.Op == lp.OpContains:
            return lit is None or lit in x
        if e.Op == lp.OpNotContains:
            return lit is None or lit not in x
        m = re.search(lit, x) is not None
        return m if e.Op == lp.OpRegexMatch else not m
    if x is None or lit is None:
        return False
    if isinstance(x, float) or isinstance(lit, float):
        x, lit = float(x), float(lit)
        if math.isnan(lit) or math.isnan(x):
            return e.Op == lp.OpNotEq
    return _cmp(e.Op, x, lit)


def distinct_rows(parts: List[Dict[str, list]], keys: List[lp.Expr], filt: lp.Expr = None) -> List[tuple]:
    """Distinct rows of the keys (plain columns or boolean expressions) over the parts, rows passing `filt`."""
    rows = set()
    for part in parts:
        n = len(next(iter(part.values())))
        for i in range(n):
            if filt is not None and not eval_bool(filt, part, i):
                continue
            rows.add(tuple(eval_bool(k, part, i) if isinstance(k, lp.BinaryExpr) else part.get(k.ColumnName, [None] * n)[i]
                           for k in keys))
    return sorted(rows, key=lambda r: tuple((x is None, x) for x in r))
