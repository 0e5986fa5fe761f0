"""Arithmetic aggregate inputs, computed group keys, int64 keys and packed dictionary keys on the general scan kernel
k_scan, against the plain reference of tests/numeric_edges.py (and against the oracle where its hash-only grouping
and its merge order cannot change the answer).

What runs here is k_scan's own work: the expression programs (vec_eval_expr / apply_arith: wrapping int64 + - *,
truncating division, zero divisors, INT64_MIN / -1, float specials, NULL rows read as 0), the hash table
(vec_slots_hash with its per-lane last-key cache, hash_find_or_insert, the packing of dictionary codes into key words
up to kMaxKeyWords) and the host's post-aggregate projection over the results.  Every plan runs under each switch
set of SWITCHES (vector lengths 128 / 256 / 1024, a ring of two stages, no pruning); with the default switches the
result statistics must show that k_scan took every row group."""
import ctypes as C
import os

import pytest

from frostdb_b200 import _lib
from frostdb_b200 import dynparquet as dp
from frostdb_b200 import logicalplan as lp
from frostdb_b200 import query
from frostdb_b200.physicalplan import GPUScan
from tests import numeric_edges as ne
from tests.test_gpu_parity import Pair
from tests.test_oracle_expressions import expr_parts, hash_key_parts, int_key_parts

pytestmark = pytest.mark.gpu

SWITCHES = [{}, {"FROSTGPU_VL": "128"}, {"FROSTGPU_VL": "1024"}, {"FROSTGPU_RING": "2"}, {"FROSTGPU_NO_PRUNE": "1"}]


@pytest.fixture(autouse=True)
def clean_switches():
    yield
    for sw in SWITCHES:
        for k in sw:
            os.environ.pop(k, None)


@pytest.fixture(scope="module")
def tables(store):
    """{name: (Pair, physical parts)}: the expression parts (sorted with negative timestamps, unsorted with the
    divisor set), int64 keys, hash-mode dictionary keys, and `value` as nullable PLAIN and CK_DICT64 chunks."""
    made = {}
    for name, parts in (("expr", list(zip(expr_parts(), (True, False)))), ("ikeys", list(zip(int_key_parts(), (True, False)))),
                        ("hkeys", [(c, False) for c in hash_key_parts()])):
        p = Pair(store, f"expressions_{name}", dp.SampleDefinitionWithFloat())
        for cols, sort in parts:
            buf = ne.write(cols, sort=sort)
            p.gt.InsertParquet(buf)
            p.ot.InsertParquet(buf)
        made[name] = (p, [ne.physical(c) for c, _ in parts])
    p = Pair(store, "expressions_enc", dp.SampleDefinition())
    enc = ne.encoded_parts(61)
    for _, _, buf in enc:
        p.gt.InsertParquet(buf)
        p.ot.InsertParquet(buf)
    made["enc"] = (p, [ne.physical(c) for _, c, _ in enc])
    yield made
    for p, _ in made.values():
        p.close()


def key_expr(k):
    return lp.Col(k) if isinstance(k, str) else k


def key_names(keys):
    return [k if isinstance(k, str) else k.Name() for k in keys]


def scan(q, filt):
    return q.Filter(filt) if filt is not None else q


def gpu_agg(p, filt, keys, aggs):
    out = []
    scan(query.NewEngine(None, p.db.TableProvider()).ScanTable(p.name), filt).Aggregate(aggs, [key_expr(k) for k in keys]) \
        .Execute(None, lambda c, r: out.append(r))
    return ne.result_map(out, key_names(keys), aggs)


def oracle_agg(p, filt, keys, aggs):
    from tests.oracle_scan import oracle_query
    out = []
    scan(oracle_query(p.oe, p.name), filt).Aggregate(aggs, [key_expr(k) for k in keys]).Execute(None, lambda c, r: out.append(r))
    return ne.result_map(out, key_names(keys), aggs)


def stats_of(p, filt, keys, aggs, kind=_lib.PLAN_AGGREGATE):
    eng, lib = p.store.engine, _lib.load()
    q, keep = GPUScan(eng, p.name, filt, kind, [key_expr(k) for k in keys], aggs).prepare()
    res = C.c_void_p()
    try:
        _lib.check(lib.fgpu_query_execute(eng.handle, q, eng.table_watermark(p.name), C.byref(res)))
        st = eng.stats(res)
        lib.fgpu_result_free(res)
    finally:
        lib.fgpu_query_free(q)
    return st


def float_minmax(aggs):
    return any(a.Func in (lp.AggFuncMin, lp.AggFuncMax) and ne.F in a.Expr.Name() for a in aggs)


def on_k_scan(st):
    return st["row_groups_runs"] == 0 and st["row_groups_tiles"] == 0


def check(tab, filt, keys, aggs, *, with_oracle=True):
    """Every switch set against the reference (and the oracle); with the default switches, k_scan took every row
    group."""
    p, phys = tab
    what = f"{p.name} filter {filt.Name() if filt is not None else None} keys {key_names(keys)} {[a.Name() for a in aggs]}"
    exp = ne.reference(phys, filt, keys, aggs)
    assert exp, what
    if with_oracle and ne.oracle_groups_exactly(keys, phys[0]) and not float_minmax(aggs):  # the oracle runs 4 threads
        ne.assert_same_result(oracle_agg(p, filt, keys, aggs), exp, aggs, what + " oracle")
    for sw in SWITCHES:
        os.environ.update(sw)
        try:
            got = gpu_agg(p, filt, keys, aggs)
        finally:
            for k in sw:
                os.environ.pop(k)
        ne.assert_same_result(got, exp, aggs, f"{what} {sw}")
    st = stats_of(p, filt, keys, aggs)
    assert st["row_groups"] > 0 and on_k_scan(st), f"{what}: row groups {st['row_groups']}, runs {st['row_groups_runs']}, tiles {st['row_groups_tiles']}"


# ---- aggregate inputs ------------------------------------------------------------------------------------------------
def test_int_aggregate_inputs(tables):
    for f in ne.expr_filters():
        for e in ne.int_expr_inputs():
            check(tables["expr"], f, ne.KEYS, ne._all4(e))


def test_eight_expression_aggregates_behind_a_computed_key(tables):
    for f in ne.expr_filters():
        check(tables["expr"], f, [ne.bucket(1000)], ne.many_int_aggs())
        check(tables["expr"], f, ["labels.a", ne.bucket(1000)], ne.many_int_aggs())


def test_int_aggregate_inputs_in_other_encodings(tables):
    """`value` as an optional PLAIN chunk and as CK_DICT64, both with NULLs (read as 0)."""
    for e in ne.int_expr_inputs():
        check(tables["enc"], None, ne.KEYS, ne._all4(e))
    check(tables["enc"], lp.Or(ne.leaf(ne.V, lp.OpLt, 0), ne.leaf(ne.T, lp.OpEq, 3)), ne.KEYS, ne._all4(lp.Mul(lp.Col(ne.V), lp.Col(ne.T))))


def test_float_aggregate_inputs(tables):
    for aggs in ne.float_expr_aggs():
        check(tables["expr"], None, ne.KEYS, aggs)


# ---- group keys ------------------------------------------------------------------------------------------------------
def test_computed_keys(tables):
    aggs = [lp.Sum(lp.Col(ne.V)), lp.Min(lp.Col(ne.V)), lp.Count(lp.Col(ne.V))]
    for keys in ne.computed_key_sets():
        check(tables["expr"], None, keys, aggs)
    check(tables["expr"], lp.Or(ne.leaf(ne.V, lp.OpLt, -1), ne.leaf(ne.T, lp.OpEq, 0)), [ne.bucket(7), "labels.b"], aggs)


def test_int64_column_keys_at_the_ends(tables):
    aggs = [lp.Sum(lp.Col(ne.T)), lp.Min(lp.Col(ne.T)), lp.Max(lp.Col(ne.T)), lp.Count(lp.Col(ne.T))]
    for keys in ([ne.V], [ne.V, "labels.a"], ["labels.b", ne.V, ne.bucket(7)]):
        check(tables["ikeys"], None, keys, aggs)
        check(tables["ikeys"], ne.leaf(ne.T, lp.OpGtEq, ne.RG + 5), keys, aggs)
    # NULL int64 keys group with 0 (the dataset holds a real 0 next to them).  The oracle prints such a group's key
    # as NULL or 0 depending on which row its merge order puts first (unpinned, DESIGN §2): reference only.
    check(tables["enc"], None, [ne.V], [lp.Count(lp.Col(ne.V)), lp.Sum(lp.Col(ne.T))], with_oracle=False)
    check(tables["enc"], None, [ne.V, "labels.a"], [lp.Count(lp.Col(ne.V)), lp.Min(lp.Col(ne.T))], with_oracle=False)


def test_packed_dictionary_keys(tables):
    aggs = [lp.Sum(lp.Col(ne.T)), lp.Max(lp.Col(ne.V)), lp.Count(lp.Col(ne.T))]
    for keys in ne.HASH_KEY_SETS:
        check(tables["hkeys"], None, keys, aggs)
    check(tables["hkeys"], ne.leaf("labels.c", lp.OpNotEq, "v004094"), ["labels.c", "labels.d"], aggs)


def test_distinct_over_int64_and_mixed_keys(tables):
    for name, keys in (("ikeys", [ne.V]), ("ikeys", [ne.V, "labels.a"]), ("hkeys", ["labels.c", "labels.d"]),
                       ("hkeys", ["labels.d"] + ne.HASH_KEY_SETS[1] + [ne.V])):
        p, phys = tables[name]
        exp = set(ne.reference(phys, None, keys, []))
        for sw in SWITCHES:
            os.environ.update(sw)
            try:
                out = []
                query.NewEngine(None, p.db.TableProvider()).ScanTable(p.name).Distinct(*[lp.Col(k) for k in keys]) \
                    .Execute(None, lambda c, r: out.append(r))
            finally:
                for k in sw:
                    os.environ.pop(k)
            got = ne.result_map(out, keys, [])
            assert set(got) == exp, f"{name} distinct {keys} {sw}: {len(got)} groups, expected {len(exp)}"
        st = stats_of(p, None, keys, [], _lib.PLAN_DISTINCT)
        assert st["row_groups"] > 0 and on_k_scan(st)


# ---- post-aggregate projection ---------------------------------------------------------------------------------------
def test_post_aggregate_projection_at_the_edges(tables):
    p, phys = tables["expr"]
    aggs = [lp.Min(lp.Col(ne.V)), lp.Max(lp.Col(ne.V)), lp.Sum(lp.Col(ne.V))]
    names = [a.Name() for a in aggs]
    mn, mx, sm = (lp.Col(n) for n in names)
    exprs = [lp.Div(mn, lp.Literal(2)), lp.Div(mn, lp.Literal(-1)), lp.Div(mx, lp.Literal(-3)), lp.Sub(mn, lp.Literal(1)),
             lp.Sub(lp.Literal(ne.I64_MIN), mx), lp.Mul(mx, lp.Literal(2)), lp.Mul(sm, mn), lp.Div(sm, lp.Literal(0)),
             lp.Div(mx, mn)]
    ref = ne.reference(phys, None, ne.KEYS, aggs)
    assert any(v[0] == ne.I64_MIN for v in ref.values()) and any(v[1] == ne.I64_MAX for v in ref.values())
    exp = ne.post_project(ref, names, exprs)
    out = []
    query.NewEngine(None, p.db.TableProvider()).ScanTable(p.name).Aggregate(aggs, [lp.Col(k) for k in ne.KEYS]) \
        .Project(*([lp.Col(k) for k in ne.KEYS] + exprs)).Execute(None, lambda c, r: out.append(r))
    got = {}
    for b in out:
        cols = [b.column(b.schema.get_field_index(n)).to_pylist() for n in ne.KEYS + [e.Name() for e in exprs]]
        for r in zip(*cols):
            got[tuple(x.decode() if isinstance(x, bytes) else x for x in r[:2])] = tuple(r[2:])
    assert got == exp
