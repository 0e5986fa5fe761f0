"""Mirror of `query/physicalplan`'s operator surface around the GPU scan.

`Build` walks the logical plan like physicalplan.Build (query/physicalplan/physicalplan.go:287-516)
and replaces the prefix TableScan [-> Filter] [-> Projection] -> Aggregation | Distinct by ONE
ScanPhysicalPlan, `GPUScan`, whose Execute hands the plan to libfrostgpu through the C-ABI and pushes
the result records into the next operator's Callback — exactly the seam the Go shim uses
(go/physicalplan_gpu.go, INTEGRATION.md).  Everything behind the aggregate (alias/avg projection,
limit) stays a host operator, as it stays a Go operator in the reference.
"""
from __future__ import annotations

import ctypes as C
import re
from typing import Callable, List, Optional

import numpy as np
import pyarrow as pa

from . import _lib
from . import logicalplan as lp


class Diagram:
    def __init__(self, details: str, child: Optional["Diagram"] = None):
        self.Details, self.Child = details, child

    def String(self) -> str:  # physicalplan.go:558-572
        s, d = self.Details, self.Child
        while d is not None:
            s += " - " + d.Details
            d = d.Child
        return s


class PhysicalPlan:
    """physicalplan.PhysicalPlan (physicalplan.go:24-30)."""
    next: Optional["PhysicalPlan"] = None

    def Callback(self, ctx, r: pa.RecordBatch) -> None: raise NotImplementedError
    def Finish(self, ctx) -> None: self.next.Finish(ctx)
    def SetNext(self, nxt: "PhysicalPlan") -> None: self.next = nxt
    def Draw(self) -> Diagram: raise NotImplementedError
    def Close(self) -> None:
        if self.next is not None:
            self.next.Close()


class OutputPlan(PhysicalPlan):
    """physicalplan.go:57-94."""

    def __init__(self):
        self.callback: Optional[Callable] = None
        self.scan: Optional["GPUScan"] = None

    def Draw(self): return Diagram("")
    def DrawString(self) -> str: return self.scan.Draw().String()
    def SetNextCallback(self, cb): self.callback = cb
    def Callback(self, ctx, r): return self.callback(ctx, r)
    def Finish(self, ctx): return None
    def Close(self): return None
    def Execute(self, ctx, pool=None): return self.scan.Execute(ctx, pool)


# ---- plan -> C-ABI ----------------------------------------------------------------------------------
class _PlanEncoder:
    """Flattens logicalplan.Expr trees into the fgpu_expr array (children before parents)."""

    def __init__(self):
        self.exprs: List[_lib.Expr] = []
        self.keep = []  # python objects the C structs point at

    def add(self, e: lp.Expr) -> int:
        x = _lib.Expr()
        x.left = x.right = -1
        if isinstance(e, lp.AliasExpr):
            return self.add(e.Expr)
        if isinstance(e, lp.Column):
            x.kind = _lib.EXPR_COLUMN
            b = e.ColumnName.encode()
            self.keep.append(b)
            x.name = b
        elif isinstance(e, lp.DynamicColumn):
            x.kind = _lib.EXPR_DYNCOLUMN
            b = e.ColumnName.encode()
            self.keep.append(b)
            x.name = b
        elif isinstance(e, lp.LiteralExpr):
            x.kind = _lib.EXPR_LITERAL
            v = e.Value
            if v is None:
                x.literal.type = _lib.SCALAR_NULL
            elif isinstance(v, bool):
                raise _lib.FrostGPUError(_lib.FGPU_ERR_UNSUPPORTED, "boolean literals are not supported on the GPU path")
            elif isinstance(v, (int, np.integer)):
                x.literal.type = _lib.SCALAR_INT64
                x.literal.i64 = int(v)
            elif isinstance(v, (float, np.floating)):
                x.literal.type = _lib.SCALAR_FLOAT64
                x.literal.f64 = float(v)
            else:
                b = v.encode() if isinstance(v, str) else bytes(v)
                buf = C.create_string_buffer(b, len(b) if b else 1)
                self.keep.append(buf)
                x.literal.type = _lib.SCALAR_STRING
                x.literal.bytes = C.addressof(buf)
                x.literal.len = len(b)
        elif isinstance(e, lp.BinaryExpr):
            l = self.add(e.Left)
            r = self.add(e.Right)
            x.kind = _lib.EXPR_BINARY
            x.op = e.Op
            x.left, x.right = l, r
            if e.Op in (lp.OpRegexMatch, lp.OpRegexNotMatch):
                # Go's regexp (RE2) semantics live on the host: filter.go:104-123 compiles the
                # pattern there.  MatchString is an unanchored search.
                pat = e.Right.Value
                rx = re.compile(pat if isinstance(pat, str) else pat.decode())

                def match(_user, ptr, n, rx=rx):
                    s = C.string_at(ptr, n).decode("utf-8", "replace") if n else ""
                    return 1 if rx.search(s) else 0

                fn = _lib.MATCH_FN(match)
                self.keep.append(fn)
                x.match = fn
        else:
            raise _lib.FrostGPUError(_lib.FGPU_ERR_UNSUPPORTED, f"expression {type(e).__name__} is not supported on the GPU path")
        self.exprs.append(x)
        return len(self.exprs) - 1


class GPUScan:
    """ScanPhysicalPlan (physicalplan.go:32-35) executing the fused prefix on the GPU."""

    def __init__(self, engine, table_name: str, filter_expr, kind: int, group_exprs, agg_exprs):
        self.engine = engine
        self.table_name = table_name
        self.filter_expr = filter_expr
        self.kind = kind
        self.group_exprs = list(group_exprs)
        self.agg_exprs = list(agg_exprs)
        self.next: Optional[PhysicalPlan] = None
        self.last_stats: Optional[dict] = None
        # computed group keys arrive as AliasExpr (sqlparse pre-projection: `(timestamp/1000)*1000 as bucket`); the
        # library names the result column after the expression, the record is renamed to the alias here
        self.rename = {g.Expr.Name(): g.AliasName for g in self.group_exprs if isinstance(g, lp.AliasExpr)}

    def SetNext(self, nxt): self.next = nxt

    def renamed(self, rec: pa.RecordBatch) -> pa.RecordBatch:
        if not self.rename:
            return rec
        return pa.RecordBatch.from_arrays(rec.columns, names=[self.rename.get(n, n) for n in rec.schema.names])

    def Draw(self) -> Diagram:
        what = ("distinct " if self.kind == _lib.PLAN_DISTINCT else "") + ",".join(a.Name() for a in self.agg_exprs)
        by = ",".join(g.Name() for g in self.group_exprs)
        det = f"GPUScan ({what}{' by ' if by and self.agg_exprs else ''}{by}"
        if self.filter_expr is not None:
            det += f" | filter {self.filter_expr.Name()}"
        det += ")"
        return Diagram(det, self.next.Draw() if self.next is not None else None)

    def _plan(self):
        enc = _PlanEncoder()
        filt = enc.add(self.filter_expr) if self.filter_expr is not None else -1
        groups = [enc.add(g) for g in self.group_exprs]
        aggs = [(a.Func, enc.add(a.Expr)) for a in self.agg_exprs]
        plan = _lib.Plan()
        tb = self.table_name.encode()
        ex = (_lib.Expr * max(len(enc.exprs), 1))(*enc.exprs)
        gb = (C.c_int32 * max(len(groups), 1))(*groups)
        ag = (_lib.Agg * max(len(aggs), 1))(*[_lib.Agg(f, e) for f, e in aggs])
        plan.table, plan.kind = tb, self.kind
        plan.n_exprs, plan.exprs = len(enc.exprs), ex
        plan.filter = filt
        plan.n_group_by, plan.group_by = len(groups), gb
        plan.n_aggs, plan.aggs = len(aggs), ag
        return plan, (enc, tb, ex, gb, ag)

    def prepare(self):
        lib = _lib.load()
        plan, keep = self._plan()
        q = C.c_void_p()
        _lib.check(lib.fgpu_query_prepare(self.engine.handle, C.byref(plan), C.byref(q)))
        return q, keep

    def Execute(self, ctx, pool=None) -> None:
        lib = _lib.load()
        tx = self.engine.table_watermark(self.table_name)  # Table.View -> DB.beginRead (table.go:731-737)
        q, keep = self.prepare()
        try:
            res = C.c_void_p()
            _lib.check(lib.fgpu_query_execute(self.engine.handle, q, tx, C.byref(res)))
            try:
                for rec in self.engine.drain(res):
                    self.next.Callback(ctx, self.renamed(rec))
                self.last_stats = self.engine.stats(res)
            finally:
                lib.fgpu_result_free(res)
        finally:
            lib.fgpu_query_free(q)
            del keep
        self.next.Finish(ctx)


# ---- host operators behind the aggregate (they stay Go in the reference) ----------------------------
def _eval_post(e: lp.Expr, r: pa.RecordBatch):
    """Evaluates a post-aggregate projection expression over a result record.
    Returns (name, pyarrow array).  Integer division truncates toward zero and a zero divisor
    yields NULL (project.go:216-218, 273-275)."""
    if isinstance(e, lp.AliasExpr):
        _, arr = _eval_post(e.Expr, r)
        return e.AliasName, arr
    if isinstance(e, lp.LiteralExpr):
        return e.Name(), pa.array([e.Value] * r.num_rows)
    if isinstance(e, lp.BinaryExpr) and lp.OpAdd <= e.Op <= lp.OpDiv:
        _, l = _eval_post(e.Left, r)
        _, rr = _eval_post(e.Right, r)
        is_float = pa.types.is_floating(l.type) or pa.types.is_floating(rr.type)
        a = np.asarray(l.fill_null(0), dtype=np.float64 if is_float else np.int64)
        b = np.asarray(rr.fill_null(0), dtype=np.float64 if is_float else np.int64)
        mask = None
        with np.errstate(all="ignore"):
            if e.Op == lp.OpAdd: out = a + b
            elif e.Op == lp.OpSub: out = a - b
            elif e.Op == lp.OpMul: out = a * b
            else:
                mask = b == 0
                if is_float:
                    out = np.where(mask, 0.0, a / np.where(mask, 1.0, b))
                else:
                    # floor division corrected toward zero; a divisor of -1 negates (INT64_MIN / -1 wraps to
                    # INT64_MIN), so no quotient leaves int64 on the way (abs(INT64_MIN) would)
                    bb = np.where(mask | (b == -1), 1, b)
                    qv = a // bb
                    qv = qv + (((a % bb) != 0) & ((a < 0) != (bb < 0)))
                    out = np.where(b == -1, np.int64(0) - a, qv).astype(np.int64)
        return e.Name(), pa.array(out, mask=mask if mask is not None and mask.any() else None)
    name = e.Name()
    idx = r.schema.get_field_index(name)
    if idx < 0:
        raise KeyError(f"column {name!r} not found in {r.schema.names}")
    return name, r.column(idx)


class Projection(PhysicalPlan):
    """Post-aggregate Projection (project.go:865-965): pass-through, alias, arithmetic."""

    def __init__(self, exprs: List[lp.Expr]):
        self.exprs = exprs

    def Draw(self):
        return Diagram("Projection (" + ", ".join(e.Name() for e in self.exprs) + ")", self.next.Draw() if self.next else None)

    def Callback(self, ctx, r: pa.RecordBatch):
        names, arrays = [], []
        for e in self.exprs:
            if isinstance(e, lp.DynamicColumn):  # dynamicProjection project.go:730-755
                for i, f in enumerate(r.schema):
                    if e.MatchColumn(f.name):
                        names.append(f.name)
                        arrays.append(r.column(i))
                continue
            if isinstance(e, lp.Column) and r.schema.get_field_index(e.ColumnName) < 0:
                continue  # plainProjection: column absent from this record
            n, a = _eval_post(e, r)
            names.append(n)
            arrays.append(a)
        if not arrays:
            return
        self.next.Callback(ctx, pa.RecordBatch.from_arrays(arrays, names=names))


class Limiter(PhysicalPlan):
    """limit.go:63-98."""

    def __init__(self, count: int):
        self.count, self.seen = count, 0

    def Draw(self):
        return Diagram(f"Limit({self.count})", self.next.Draw() if self.next else None)

    def Callback(self, ctx, r):
        if self.seen >= self.count:
            return
        take = min(r.num_rows, self.count - self.seen)
        self.seen += take
        self.next.Callback(ctx, r.slice(0, take))


def Build(engine, plan: lp.LogicalPlan, scan_factory=None) -> OutputPlan:
    """Pattern-matches the GPU-executable prefix and chains the remaining host operators."""
    scan_factory = scan_factory or GPUScan
    nodes = plan.chain()
    if not nodes or nodes[0].TableScan is None:
        raise _lib.FrostGPUError(_lib.FGPU_ERR_INVALID, "plan must start with a TableScan")
    scan = nodes[0].TableScan
    i = 1
    filter_expr = scan.Filter
    while i < len(nodes) and nodes[i].Filter is not None:  # FilterPushDown: filters fold into the scan
        filter_expr = nodes[i].Filter.Expr if filter_expr is None else lp.And(filter_expr, nodes[i].Filter.Expr)
        i += 1
    def passthrough(proj) -> bool:
        # Projection feeding the aggregate (sqlparse pre-projection): plain / dynamic columns and the
        # arithmetic the aggregate expressions repeat; the fused scan reads what it needs itself.
        def ok(e):
            if isinstance(e, lp.AliasExpr):  # `(timestamp / 1000) * 1000 as timestamp_bucket`: a computed group key
                return isinstance(e.Expr, lp.BinaryExpr) and ok(e.Expr)
            if isinstance(e, (lp.Column, lp.DynamicColumn)):
                return True
            return isinstance(e, lp.BinaryExpr) and lp.OpAdd <= e.Op <= lp.OpDiv and ok_operand(e.Left) and ok_operand(e.Right)

        def ok_operand(e):
            return isinstance(e, (lp.Column, lp.LiteralExpr)) or ok(e)
        return all(ok(e) for e in proj.Exprs)

    aliases = {}
    if (i + 1 < len(nodes) and nodes[i].Projection is not None and nodes[i + 1].Aggregation is not None
            and passthrough(nodes[i].Projection)):
        aliases = {e.AliasName: e for e in nodes[i].Projection.Exprs if isinstance(e, lp.AliasExpr)}
        i += 1
    gpu: Optional[GPUScan] = None
    if i < len(nodes) and nodes[i].Aggregation is not None:
        a = nodes[i].Aggregation
        # a group column that names an aliased pre-projection is that expression (computed group key)
        group_exprs = [aliases.get(g.ColumnName, g) if isinstance(g, lp.Column) else g for g in a.GroupExprs]
        gpu = scan_factory(engine, scan.TableName, filter_expr, _lib.PLAN_AGGREGATE, group_exprs, a.AggExprs)
        i += 1
    elif i + 1 < len(nodes) and nodes[i].Projection is not None and nodes[i + 1].Distinct is not None:
        d = nodes[i + 1].Distinct
        gpu = scan_factory(engine, scan.TableName, filter_expr, _lib.PLAN_DISTINCT, d.Exprs, [])
        i += 2
    elif (i < len(nodes) and nodes[i].Projection is not None
          and all(isinstance(e, (lp.Column, lp.DynamicColumn)) for e in nodes[i].Projection.Exprs)):
        # TableScan -> Filter -> Projection(columns): compacted rows (PredicateFilter + Projection)
        gpu = scan_factory(engine, scan.TableName, filter_expr, _lib.PLAN_FILTER, nodes[i].Projection.Exprs, [])
        i += 1
    else:
        raise _lib.FrostGPUError(_lib.FGPU_ERR_UNSUPPORTED,
                                 "the GPU engine covers TableScan[->Filter]->Aggregation|Distinct|Projection(columns); "
                                 "keep this plan on the Go operators")
    out = OutputPlan()
    out.scan = gpu
    prev = gpu
    for n in nodes[i:]:
        if n.Projection is not None:
            op: PhysicalPlan = Projection(n.Projection.Exprs)
        elif n.Limit is not None:
            op = Limiter(int(n.Limit.Expr.Value))
        else:
            raise _lib.FrostGPUError(_lib.FGPU_ERR_UNSUPPORTED, "operator after the aggregate is not supported")
        prev.SetNext(op)
        prev = op
    prev.SetNext(out)
    return out
