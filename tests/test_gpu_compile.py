"""Every refusal of the plan compiler (compile() in engine.cpp, with compile_filter and compile_agg_expr) that a plan
can reach through fgpu_query_execute, asserted by error code and message, and the order in which the checks fire
where one plan trips two of them.

Two refusals cannot be reached through the ABI:
- "filter expression too large" (more than kMaxFilterProg = 96 program bytes): at most kMaxLeaves = 32 leaves make
  at most 63 bytes, and "too many predicate leaves" fires first.
- "too many projected columns" (a rows plan with more than kMaxOut = 40 columns): kMaxKeys is also 40, and
  "too many group-by columns" fires first.

Tables: `main` has two parts of 100 rows each.  Part 0 holds `only0` and `labels.b`; part 1 holds neither, but
holds a column literally named "value + 1".  Their timestamps do not overlap, so a filter on timestamp can
prune either part by its statistics.  `types` changes the type of `x` between its parts.  `odd` holds an int32
and a uint64 column.  `wide` has 49 labels columns."""
import ctypes as C
import os

import numpy as np
import pyarrow as pa
import pytest

from frostdb_b200 import _lib
from frostdb_b200 import dynparquet as dp
from frostdb_b200 import logicalplan as lp
from frostdb_b200.physicalplan import GPUScan

pytestmark = pytest.mark.gpu

INVALID, UNSUPPORTED, NOT_FOUND = _lib.FGPU_ERR_INVALID, _lib.FGPU_ERR_UNSUPPORTED, _lib.FGPU_ERR_NOT_FOUND
AGG, DISTINCT = _lib.PLAN_AGGREGATE, _lib.PLAN_DISTINCT
N = 100
WIDE = 49  # kMaxSlots + 1
V, F, T, A = lp.Col("value"), lp.Col("floatvalue"), lp.Col("timestamp"), lp.Col("labels.a")


def schema(**types):
    cols = [dp.ColumnDefinition("labels", dp.TYPE_STRING, nullable=True, dynamic=True, rle_dictionary=True)]
    cols += [dp.ColumnDefinition(n, t, nullable=True) for n, t in types.items()]
    return dp.Schema("compile", cols, [dp.SortingColumn("timestamp")])


def labels(card):
    return (np.arange(N, dtype=np.int32) % card, [f"v{i}" for i in range(card)])


@pytest.fixture(scope="module")
def tables(store):
    eng = store.engine
    names = {k: f"compile_{k}" for k in ("main", "types", "odd", "wide")}
    for n in names.values():
        eng.drop_table(n)
    ts = np.arange(N, dtype=np.int64)
    s = schema(timestamp=dp.TYPE_INT64, value=dp.TYPE_INT64, floatvalue=dp.TYPE_DOUBLE, only0=dp.TYPE_INT64,
               **{"value + 1": dp.TYPE_INT64})
    eng.put_parquet(names["main"], dp.write_part(s, {"labels.a": labels(4), "labels.b": labels(3), "timestamp": ts,
                                                    "value": ts % 7, "floatvalue": ts / 4.0, "only0": ts}))
    eng.put_parquet(names["main"], dp.write_part(s, {"labels.a": labels(5), "timestamp": 1000 + ts, "value": ts % 5,
                                                    "floatvalue": ts / 8.0, "value + 1": ts}))
    eng.put_parquet(names["types"], dp.write_part(schema(timestamp=dp.TYPE_INT64, x=dp.TYPE_INT64), {"timestamp": ts, "x": ts}))
    eng.put_parquet(names["types"], dp.write_part(schema(timestamp=dp.TYPE_INT64, x=dp.TYPE_DOUBLE), {"timestamp": ts, "x": ts * 0.5}))
    s = schema(timestamp=dp.TYPE_INT64, value=dp.TYPE_INT64, i32=dp.TYPE_INT64, u64=dp.TYPE_INT64)
    eng.put_parquet(names["odd"], dp.write_part(s, {"timestamp": ts, "value": ts, "i32": pa.array(ts.astype(np.int32)),
                                                   "u64": pa.array(ts.astype(np.uint64))}, sort=False))
    wide = {f"labels.l{i:02d}": labels(2) for i in range(WIDE)}
    eng.put_parquet(names["wide"], dp.write_part(schema(value=dp.TYPE_INT64), dict(wide, value=ts), sort=False))
    yield names
    for n in names.values():
        eng.drop_table(n)


def execute(store, table, filt=None, groups=(), aggs=(), kind=AGG, patch=None):
    """Runs the plan once; returns None when it executes, else (error code, message)."""
    eng, lib = store.engine, _lib.load()
    plan, keep = GPUScan(eng, table, filt, kind, list(groups), list(aggs))._plan()
    if patch:
        patch(plan)
    q, res = C.c_void_p(), C.c_void_p()
    _lib.check(lib.fgpu_query_prepare(eng.handle, C.byref(plan), C.byref(q)))
    try:
        _lib.check(lib.fgpu_query_execute(eng.handle, q, eng.table_watermark(table), C.byref(res)))
        list(eng.drain(res))
        lib.fgpu_result_free(res)
        return None
    except _lib.FrostGPUError as e:
        return e.code, e.msg
    finally:
        lib.fgpu_query_free(q)
        del keep


def nest(depth):
    """value + (value + (...)): an operand stack `depth` values deep."""
    e = V
    for _ in range(depth - 1):
        e = lp.Add(V, e)
    return e


def long_chain(e, n=25):
    """((e + 1) + 1) ...: 2n + 1 program ops at stack depth 2, over kMaxProg = 48 for n = 25."""
    for _ in range(n):
        e = lp.Add(e, lp.Literal(1))
    return e


def eq(col, v):
    return lp.BinaryExpr(lp.Col(col), lp.OpEq, lp.Literal(v))


def drop_matcher(plan):
    for i in range(plan.n_exprs):
        if plan.exprs[i].op == lp.OpRegexMatch:
            plan.exprs[i].match = _lib.MATCH_FN()


C_ = lp.Count(V)
# (table, plan, expected code, expected message substring)
REFUSALS = {
    # columns and group keys
    "changes_type": ("types", dict(aggs=[C_]), UNSUPPORTED, "column x changes type between parts"),
    "unread_type": ("odd", dict(aggs=[lp.Sum(lp.Col("i32"))]), UNSUPPORTED, "column i32 has a type the GPU engine does not read"),
    "too_many_columns": ("wide", dict(filt=lp.Or(*[eq(f"labels.l{i:02d}", "v0") for i in range(WIDE)]), aggs=[C_]),
                         UNSUPPORTED, "query touches too many columns"),
    "key_shadows_column": ("main", dict(groups=[lp.Add(V, lp.Literal(1))], aggs=[C_]), UNSUPPORTED,
                           "computed group key shadows a column: value + 1"),
    "literal_key": ("main", dict(groups=[lp.Literal(3)], aggs=[C_]), UNSUPPORTED,
                    "this group-by expression is not supported on the GPU path"),
    "distinct_computed_key": ("main", dict(groups=[lp.Mul(V, lp.Literal(2))], kind=DISTINCT), UNSUPPORTED,
                              "this group-by expression is not supported on the GPU path"),
    "too_many_keys": ("wide", dict(groups=[lp.DynCol("labels")], aggs=[C_]), UNSUPPORTED, "too many group-by columns"),
    # filter program and leaves
    "filter_not_binary": ("main", dict(filt=V, aggs=[C_]), UNSUPPORTED, "unsupported boolean expression"),
    "filter_arithmetic": ("main", dict(filt=lp.Add(V, lp.Literal(1)), aggs=[C_]), UNSUPPORTED, "unsupported filter operator +"),
    "literal_on_left": ("main", dict(filt=lp.BinaryExpr(lp.Literal(1), lp.OpEq, V), aggs=[C_]), INVALID,
                        "left side of binary expression must be a column"),
    "column_on_right": ("main", dict(filt=V.Eq(T), aggs=[C_]), INVALID, "right side of binary expression must be a literal"),
    "regex_without_matcher": ("main", dict(filt=A.RegexMatch("v1"), aggs=[C_], patch=drop_matcher), INVALID,
                              "regex leaf without a matcher"),
    "too_many_leaves": ("wide", dict(filt=lp.And(*[eq(f"labels.l{i:02d}", "v0") for i in range(33)]), aggs=[C_]),
                        UNSUPPORTED, "too many predicate leaves"),
    "filter_too_deep": ("main", dict(filt=lp.Or(*[V.Eq(lp.Literal(i)) for i in range(31)]), aggs=[C_]), UNSUPPORTED,
                        "filter expression too deep"),
    "dict_vs_int": ("main", dict(filt=A.Eq(lp.Literal(5)), aggs=[C_]), UNSUPPORTED,
                    "dictionary column compared with a non-string literal"),
    "dict_ordering": ("main", dict(filt=A.Lt(lp.Literal("v1")), aggs=[C_]), INVALID, "unsupported operator: <"),
    "numeric_regex": ("main", dict(filt=V.RegexMatch("1"), aggs=[C_]), UNSUPPORTED, "operator =~ on a numeric column"),
    "numeric_contains": ("main", dict(filt=V.Contains("1"), aggs=[C_]), UNSUPPORTED, "operator contains on a numeric column"),
    "numeric_vs_string": ("main", dict(filt=V.Eq(lp.Literal("1")), aggs=[C_]), UNSUPPORTED,
                          "numeric column compared with a string literal"),
    # residency
    "column_image_error": ("odd", dict(aggs=[lp.Sum(lp.Col("u64"))]), UNSUPPORTED, "column u64: uint64 columns are not supported"),
    # aggregates
    "too_many_aggs": ("main", dict(aggs=[lp.Avg(V)] * 9), UNSUPPORTED, "too many aggregates"),
    "avg": ("main", dict(aggs=[lp.Avg(V)]), UNSUPPORTED, "aggregate function not supported on the GPU path: avg"),
    "agg_column_absent": ("main", dict(aggs=[lp.Sum(lp.Col("nosuch"))]), NOT_FOUND, 'aggregate field(s) not found ["nosuch"]'),
    "agg_over_dict": ("main", dict(aggs=[lp.Sum(A)]), UNSUPPORTED, "aggregation over a non-numeric column: labels.a"),
    "agg_string_literal": ("main", dict(aggs=[lp.Sum(lp.Add(V, lp.Literal("x")))]), UNSUPPORTED,
                           "non-numeric literal in arithmetic expression"),
    "agg_comparison": ("main", dict(aggs=[lp.Sum(V.Eq(lp.Literal(1)))]), UNSUPPORTED, "unsupported aggregate expression"),
    "agg_mixes_types": ("main", dict(aggs=[lp.Sum(lp.Add(V, F))]), UNSUPPORTED, "arithmetic mixes int64 and float64 columns"),
    "agg_column_in_some_parts": ("main", dict(aggs=[lp.Sum(lp.Col("only0"))]), NOT_FOUND,
                                 'aggregate field(s) not found ["only0"]'),
    "agg_too_large": ("main", dict(aggs=[lp.Sum(long_chain(V))]), UNSUPPORTED, "aggregate expressions too large"),
    "agg_too_deep": ("main", dict(aggs=[lp.Sum(nest(4))]), UNSUPPORTED, "aggregate expression nests too deeply for the GPU path"),
    # group keys and table shape
    "key_expr_column_absent": ("main", dict(groups=[lp.Add(lp.Col("nosuch"), lp.Literal(1))], aggs=[C_]), NOT_FOUND,
                               'aggregate field(s) not found ["nosuch"]'),
    "key_expr_over_dict": ("main", dict(groups=[lp.Add(A, lp.Literal(1))], aggs=[C_]), UNSUPPORTED,
                           "aggregation over a non-numeric column: labels.a"),
    "key_expr_float": ("main", dict(groups=[lp.Add(F, lp.Literal(1))], aggs=[C_]), UNSUPPORTED,
                       "float64 group-by expressions are not supported"),
    "key_expr_too_large": ("main", dict(groups=[long_chain(V)], aggs=[C_]), UNSUPPORTED, "group-by expression too large"),
    "key_expr_too_deep": ("main", dict(groups=[nest(4)], aggs=[C_]), UNSUPPORTED,
                          "group-by expression nests too deeply for the GPU path"),
    "key_expr_column_in_some_parts": ("main", dict(groups=[lp.Add(lp.Col("only0"), lp.Literal(1))], aggs=[C_]), NOT_FOUND,
                                      "group-by expression column not found: only0"),
    "float_key": ("main", dict(groups=[F], aggs=[C_]), UNSUPPORTED, "float64 group-by columns are not supported"),
    "key_too_wide": ("main", dict(groups=[lp.Sub(V, lp.Literal(k)) for k in range(1, 8)], aggs=[C_]), UNSUPPORTED,
                     "group key wider than the packed-key limit"),
}

# Plans that trip two checks; the comment names the order each case pins.
PRECEDENCE = {
    # the key count is checked before any key column takes a slot (49 key columns would also be too many slots)
    "key_count_before_slots": REFUSALS["too_many_keys"],
    # column types are resolved before anything else, even for columns the plan does not name
    "types_before_filter": ("types", dict(filt=V.Eq(lp.Literal("1")), aggs=[lp.Sum(lp.Col("nosuch"))]), UNSUPPORTED,
                            "column x changes type between parts"),
    # slots are resolved before the filter is compiled (49 leaves would also be too many)
    "slots_before_leaves": REFUSALS["too_many_columns"],
    # the leaf count is checked while compiling, before the depth of the program (33 ANDs are also too deep)
    "leaves_before_depth": REFUSALS["too_many_leaves"],
    # the program depth is checked before the leaves' operand types
    "filter_depth_before_leaf_types": ("main", dict(filt=lp.Or(*[V.Eq(lp.Literal(str(i))) for i in range(31)]), aggs=[C_]),
                                       UNSUPPORTED, "filter expression too deep"),
    # leaf operand types are checked before any column is made resident
    "leaf_types_before_residency": ("odd", dict(filt=V.Eq(lp.Literal("1")), aggs=[lp.Sum(lp.Col("u64"))]), UNSUPPORTED,
                                    "numeric column compared with a string literal"),
    # residency comes before the aggregates
    "residency_before_aggs": ("odd", dict(aggs=[lp.Sum(lp.Col("u64")), lp.Sum(lp.Add(lp.Col("value"), lp.Literal("x")))]),
                              UNSUPPORTED, "column u64: uint64 columns are not supported"),
    # the aggregate count is checked before any aggregate function
    "agg_count_before_func": REFUSALS["too_many_aggs"],
    # int64/float64 mixing is checked before the aggregate's columns are looked up in each row group
    "agg_mix_before_column_check": ("main", dict(aggs=[lp.Sum(lp.Add(lp.Col("only0"), F))]), UNSUPPORTED,
                                    "arithmetic mixes int64 and float64 columns"),
    # each aggregate's columns are looked up before the total program size is checked
    "agg_column_check_before_size": ("main", dict(aggs=[lp.Sum(long_chain(V)), lp.Sum(lp.Col("only0"))]), NOT_FOUND,
                                     'aggregate field(s) not found ["only0"]'),
    # ... and before any aggregate's depth is checked
    "agg_column_check_before_depth": ("main", dict(aggs=[lp.Sum(nest(4)), lp.Sum(lp.Col("only0"))]), NOT_FOUND,
                                      'aggregate field(s) not found ["only0"]'),
    # the total size is checked before the depth
    "agg_size_before_depth": ("main", dict(aggs=[lp.Sum(nest(4)), lp.Sum(long_chain(V))]), UNSUPPORTED,
                              "aggregate expressions too large"),
    # aggregates are compiled before the group keys
    "aggs_before_keys": ("main", dict(groups=[F], aggs=[lp.Sum(nest(4))]), UNSUPPORTED,
                         "aggregate expression nests too deeply for the GPU path"),
    # a computed key: float64 before size
    "key_float_before_size": ("main", dict(groups=[long_chain(F)], aggs=[C_]), UNSUPPORTED,
                              "float64 group-by expressions are not supported"),
    # ... size before depth
    "key_size_before_depth": ("main", dict(groups=[long_chain(nest(4), 23)], aggs=[C_]), UNSUPPORTED,
                              "group-by expression too large"),
    # ... depth before the row-group column check (the opposite of the aggregates' order)
    "key_depth_before_column_check": ("main", dict(groups=[lp.Add(lp.Col("only0"), lp.Add(V, lp.Add(V, V)))], aggs=[C_]),
                                      UNSUPPORTED, "group-by expression nests too deeply for the GPU path"),
    # keys are checked in order: a float64 column key before a later computed key
    "keys_in_order": ("main", dict(groups=[F, nest(4)], aggs=[C_]), UNSUPPORTED, "float64 group-by columns are not supported"),
}


@pytest.mark.parametrize("case", REFUSALS)
def test_refusal(store, tables, case):
    table, plan, code, msg = REFUSALS[case]
    err = execute(store, tables[table], **plan)
    assert err is not None and err[0] == code and msg in err[1], err


@pytest.mark.parametrize("case", PRECEDENCE)
def test_precedence(store, tables, case):
    table, plan, code, msg = PRECEDENCE[case]
    err = execute(store, tables[table], **plan)
    assert err is not None and err[0] == code and msg in err[1], err


def test_column_check_sees_only_kept_row_groups(store, tables):
    """A column that only the pruned part lacks is in every row group the scan reads."""
    plan = dict(filt=T.Lt(lp.Literal(500)), aggs=[lp.Sum(lp.Col("only0"))])
    assert execute(store, tables["main"], **plan) is None
    os.environ["FROSTGPU_NO_PRUNE"] = "1"
    try:
        assert execute(store, tables["main"], **plan)[0] == NOT_FOUND
    finally:
        os.environ.pop("FROSTGPU_NO_PRUNE")


def test_unnamed_columns_are_not_checked(store, tables):
    """A column of an unreadable type refuses only the plans that name it."""
    assert execute(store, tables["odd"], aggs=[lp.Sum(V)]) is None
