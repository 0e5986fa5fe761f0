"""Mirror of FrostDB's `query/logicalplan` surface needed by the scan->filter->aggregate path.

Same names and argument meaning as the Go package (query/logicalplan/expr.go, builder.go,
logicalplan.go) so plans read like the reference's: `Col("labels.job").Eq(Literal("api"))`,
`Sum(Col("value"))`, `DynCol("labels")`, `And(...)`, `Builder.Scan(...).Filter(...).Aggregate(...)`.
The Go host keeps using the real package; this mirror exists because no Go toolchain is available
here and the tests drive the C-ABI from Python.
"""
from __future__ import annotations

import dataclasses
from typing import List, Optional, Sequence

from . import _lib

Op = int
OpEq, OpNotEq, OpLt, OpLtEq, OpGt, OpGtEq = _lib.OP_EQ, _lib.OP_NOT_EQ, _lib.OP_LT, _lib.OP_LT_EQ, _lib.OP_GT, _lib.OP_GT_EQ
OpRegexMatch, OpRegexNotMatch, OpAnd, OpOr = _lib.OP_REGEX_MATCH, _lib.OP_REGEX_NOT_MATCH, _lib.OP_AND, _lib.OP_OR
OpAdd, OpSub, OpMul, OpDiv = _lib.OP_ADD, _lib.OP_SUB, _lib.OP_MUL, _lib.OP_DIV
OpContains, OpNotContains = _lib.OP_CONTAINS, _lib.OP_NOT_CONTAINS

_OP_STR = {OpEq: "==", OpNotEq: "!=", OpLt: "<", OpLtEq: "<=", OpGt: ">", OpGtEq: ">=", OpRegexMatch: "=~",
           OpRegexNotMatch: "!~", OpAnd: "&&", OpOr: "||", OpAdd: "+", OpSub: "-", OpMul: "*", OpDiv: "/",
           OpContains: "contains", OpNotContains: "not contains"}

AggFuncSum, AggFuncMin, AggFuncMax, AggFuncCount, AggFuncAvg = _lib.AGG_SUM, _lib.AGG_MIN, _lib.AGG_MAX, _lib.AGG_COUNT, _lib.AGG_AVG
AggFuncUnique = _lib.AGG_UNIQUE
_AGG_STR = {AggFuncSum: "sum", AggFuncMin: "min", AggFuncMax: "max", AggFuncCount: "count", AggFuncAvg: "avg",
            AggFuncUnique: "unique"}


class Expr:
    def Name(self) -> str:  # noqa: N802 (Go names on purpose)
        raise NotImplementedError

    def MatchColumn(self, column: str) -> bool:  # noqa: N802
        return self.Name() == column

    def Computed(self) -> bool:  # noqa: N802
        return False

    def ColumnsUsedExprs(self) -> List["Expr"]:  # noqa: N802
        return []

    def Alias(self, alias: str) -> "AliasExpr":  # noqa: N802
        return AliasExpr(self, alias)

    def __str__(self) -> str:
        return self.Name()


@dataclasses.dataclass(eq=False)
class Column(Expr):
    ColumnName: str

    def Name(self) -> str:
        return self.ColumnName

    def ColumnsUsedExprs(self):
        return [self]

    def Eq(self, e: Expr): return BinaryExpr(self, OpEq, e)
    def NotEq(self, e: Expr): return BinaryExpr(self, OpNotEq, e)
    def Gt(self, e: Expr): return BinaryExpr(self, OpGt, e)
    def GtEq(self, e: Expr): return BinaryExpr(self, OpGtEq, e)
    def Lt(self, e: Expr): return BinaryExpr(self, OpLt, e)
    def LtEq(self, e: Expr): return BinaryExpr(self, OpLtEq, e)
    def RegexMatch(self, pattern: str): return BinaryExpr(self, OpRegexMatch, Literal(pattern))
    def RegexNotMatch(self, pattern: str): return BinaryExpr(self, OpRegexNotMatch, Literal(pattern))
    def Contains(self, pattern: str): return BinaryExpr(self, OpContains, Literal(pattern))
    def ContainsNot(self, pattern: str): return BinaryExpr(self, OpNotContains, Literal(pattern))


@dataclasses.dataclass(eq=False)
class DynamicColumn(Expr):
    ColumnName: str

    def Name(self) -> str:
        return self.ColumnName

    def MatchColumn(self, column: str) -> bool:  # expr.go:564
        return column.startswith(self.ColumnName + ".")

    def ColumnsUsedExprs(self):
        return [self]


@dataclasses.dataclass(eq=False)
class LiteralExpr(Expr):
    Value: object  # None, int, float, str, bytes

    def Name(self) -> str:
        v = self.Value
        if v is None:
            return "null"
        if isinstance(v, bytes):
            return v.decode("utf-8", "replace")
        if isinstance(v, float):
            return "%g" % v
        return str(v)


@dataclasses.dataclass(eq=False)
class BinaryExpr(Expr):
    Left: Expr
    Op: int
    Right: Expr

    def Name(self) -> str:
        return f"{self.Left.Name()} {_OP_STR[self.Op]} {self.Right.Name()}"

    def Computed(self) -> bool:
        return True

    def ColumnsUsedExprs(self):
        return self.Left.ColumnsUsedExprs() + self.Right.ColumnsUsedExprs()


@dataclasses.dataclass(eq=False)
class AggregationFunction(Expr):
    Func: int
    Expr: Expr

    def Name(self) -> str:  # expr.go:700
        return f"{_AGG_STR[self.Func]}({self.Expr.Name()})"

    def ColumnsUsedExprs(self):
        return self.Expr.ColumnsUsedExprs()


@dataclasses.dataclass(eq=False)
class AliasExpr(Expr):
    Expr: Expr
    AliasName: str

    def Name(self) -> str:
        return self.AliasName

    def Computed(self) -> bool:
        return self.Expr.Computed()

    def ColumnsUsedExprs(self):
        return self.Expr.ColumnsUsedExprs()


def Col(name: str) -> Column: return Column(name)
def DynCol(name: str) -> DynamicColumn: return DynamicColumn(name)
def Cols(*names: str) -> List[Expr]: return [Col(n) for n in names]
def Literal(v) -> LiteralExpr: return LiteralExpr(v)


def _fold(exprs: Sequence[Expr], op: int) -> Expr:  # computeBinaryExpr, expr.go:489-516
    exprs = [e for e in exprs if e is not None]
    if not exprs:
        raise ValueError("no expressions")
    if len(exprs) == 1:
        return exprs[0]
    return BinaryExpr(exprs[0], op, _fold(exprs[1:], op))


def And(*exprs: Expr) -> Expr: return _fold(exprs, OpAnd)
def Or(*exprs: Expr) -> Expr: return _fold(exprs, OpOr)
def Add(l: Expr, r: Expr): return BinaryExpr(l, OpAdd, r)
def Sub(l: Expr, r: Expr): return BinaryExpr(l, OpSub, r)
def Mul(l: Expr, r: Expr): return BinaryExpr(l, OpMul, r)
def Div(l: Expr, r: Expr): return BinaryExpr(l, OpDiv, r)
def Sum(e: Expr): return AggregationFunction(AggFuncSum, e)
def Min(e: Expr): return AggregationFunction(AggFuncMin, e)
def Max(e: Expr): return AggregationFunction(AggFuncMax, e)
def Count(e: Expr): return AggregationFunction(AggFuncCount, e)
def Avg(e: Expr): return AggregationFunction(AggFuncAvg, e)
def Unique(e: Expr): return AggregationFunction(AggFuncUnique, e)


# ---- logical plan nodes (logicalplan.go:17-29) ----------------------------------------------------
@dataclasses.dataclass
class TableScan:
    TableProvider: object
    TableName: str
    Filter: Optional[Expr] = None  # set by FilterPushDown (optimize.go:81-105)


@dataclasses.dataclass
class Filter:
    Expr: Expr


@dataclasses.dataclass
class Projection:
    Exprs: List[Expr]


@dataclasses.dataclass
class Distinct:
    Exprs: List[Expr]


@dataclasses.dataclass
class Aggregation:
    AggExprs: List[AggregationFunction]
    GroupExprs: List[Expr]


@dataclasses.dataclass
class Limit:
    Expr: Expr


@dataclasses.dataclass
class LogicalPlan:
    Input: Optional["LogicalPlan"] = None
    TableScan: Optional[TableScan] = None
    Filter: Optional[Filter] = None
    Projection: Optional[Projection] = None
    Distinct: Optional[Distinct] = None
    Aggregation: Optional[Aggregation] = None
    Limit: Optional[Limit] = None

    def chain(self) -> List["LogicalPlan"]:
        """Nodes from the scan (innermost) outwards."""
        out, p = [], self
        while p is not None:
            out.append(p)
            p = p.Input
        return list(reversed(out))


class Builder:
    """logicalplan.Builder (builder.go:10-266)."""

    def __init__(self, plan: Optional[LogicalPlan] = None):
        self.plan = plan

    def Scan(self, provider, table_name: str) -> "Builder":
        return Builder(LogicalPlan(TableScan=TableScan(provider, table_name)))

    def Filter(self, expr: Optional[Expr]) -> "Builder":
        if expr is None:
            return self
        return Builder(LogicalPlan(Input=self.plan, Filter=Filter(expr)))

    def Project(self, *exprs: Expr) -> "Builder":
        return Builder(LogicalPlan(Input=self.plan, Projection=Projection(list(exprs))))

    def Distinct(self, *exprs: Expr) -> "Builder":  # builder.go:117-134: Projection then Distinct
        if not exprs:
            return self
        return Builder(LogicalPlan(Input=LogicalPlan(Input=self.plan, Projection=Projection(list(exprs))),
                                   Distinct=Distinct(list(exprs))))

    def Limit(self, expr: Optional[Expr]) -> "Builder":
        if expr is None:
            return self
        return Builder(LogicalPlan(Input=self.plan, Limit=Limit(expr)))

    def Aggregate(self, agg_exprs: Sequence[AggregationFunction], group_exprs: Sequence[Expr]) -> "Builder":
        """builder.go:152-203.  Avg(x) is resolved to Sum(x), Count(x) and a post-aggregate
        projection Div(Sum, Count) aliased to the Avg's name (resolveAggregation builder.go:205-238);
        without an Avg the plan is the bare Aggregation."""
        resolved: List[AggregationFunction] = []
        project: List[Expr] = []
        needs_post_processing = False
        for a in agg_exprs:
            if a.Func == AggFuncAvg:
                s, c = Sum(a.Expr), Count(a.Expr)
                resolved += [s, c]
                project.append(Div(s, c).Alias(a.Name()))
                needs_post_processing = True
            else:
                resolved.append(a)
                project.append(a)
        if not needs_post_processing:
            return Builder(LogicalPlan(Input=self.plan, Aggregation=Aggregation(list(agg_exprs), list(group_exprs))))
        return Builder(LogicalPlan(
            Input=LogicalPlan(Input=self.plan, Aggregation=Aggregation(resolved, list(group_exprs))),
            Projection=Projection(list(group_exprs) + project)))

    def Build(self) -> LogicalPlan:
        if self.plan is None:
            raise ValueError("empty plan")
        return self.plan
