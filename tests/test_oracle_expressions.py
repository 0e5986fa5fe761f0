"""The CPU oracle (1 and 4 worker threads) against the plain reference of tests/numeric_edges.py on arithmetic aggregate
inputs (int64 edges, zero divisors, INT64_MIN / -1, float specials and NULL rows), computed group keys (time buckets
over negative timestamps, zero-divisor groups), int64 keys at the ends of int64, and dictionary keys that pack into
several hash-key words."""
import pytest

from frostdb_b200 import dynparquet as dp
from frostdb_b200 import logicalplan as lp
from tests import numeric_edges as ne
from tests.oracle_scan import OracleEngine, OracleTableHandle, oracle_query

N_PART = ne.RG * len(ne.INT_CHUNKS)


def expr_parts():
    return [ne.expr_part(31, sort=True, t0=-N_PART // 2), ne.expr_part(32, sort=False, part=1)]


def int_key_parts():
    return [ne.int_key_part(41, sort=True), ne.int_key_part(42, sort=False, t0=10 * ne.RG)]


def hash_key_parts():
    return [ne.hash_key_part(51), ne.hash_key_part(52, t0=10 * ne.RG)]


@pytest.fixture(scope="module")
def tables():
    """Every dataset in the oracle at 1 and 4 threads: {threads: engine}, {table: physical parts}."""
    tabs = {"expr": [(c, ne.write(c, sort=s)) for c, s in zip(expr_parts(), (True, False))],
            "ikeys": [(c, ne.write(c, sort=s)) for c, s in zip(int_key_parts(), (True, False))],
            "hkeys": [(c, ne.write(c, sort=False)) for c in hash_key_parts()],
            "enc": [(c, b) for _, c, b in ne.encoded_parts(61)]}
    engines = {}
    for threads in (1, 4):
        eng = OracleEngine(threads=threads)
        for name, parts in tabs.items():
            t = OracleTableHandle(eng, name, dp.SampleDefinitionWithFloat())
            for _, buf in parts:
                t.InsertParquet(buf)
        engines[threads] = eng
    yield engines, {name: [ne.physical(c) for c, _ in parts] for name, parts in tabs.items()}
    for eng in engines.values():
        eng.close()


def key_expr(k):
    return lp.Col(k) if isinstance(k, str) else k


def key_names(keys):
    return [k if isinstance(k, str) else k.Name() for k in keys]


def float_nan_minmax(aggs):
    """Min / Max over a float input that may hold NaN: the oracle's merge order at 4 threads decides those."""
    return any(a.Func in (lp.AggFuncMin, lp.AggFuncMax) and ne.F in a.Expr.Name() for a in aggs)


def check(eng, phys, table, filt, keys, aggs, what=""):
    if not ne.oracle_groups_exactly(keys, phys[table][0]):
        return
    out = []
    q = oracle_query(eng, table)
    if filt is not None:
        q = q.Filter(filt)
    q.Aggregate(aggs, [key_expr(k) for k in keys]).Execute(None, lambda c, r: out.append(r))
    got = ne.result_map(out, key_names(keys), aggs)
    exp = ne.reference(phys[table], filt, keys, aggs)
    ne.assert_same_result(got, exp, aggs, f"{what} {table} filter {filt.Name() if filt is not None else None} keys {key_names(keys)}")


@pytest.mark.parametrize("threads", [1, 4])
def test_int_aggregate_inputs(tables, threads):
    engines, phys = tables
    for f in ne.expr_filters():
        for e in ne.int_expr_inputs():
            check(engines[threads], phys, "expr", f, ne.KEYS, ne._all4(e))
        check(engines[threads], phys, "expr", f, [ne.bucket(1000)], ne.many_int_aggs())


@pytest.mark.parametrize("threads", [1, 4])
def test_int_aggregate_inputs_in_other_encodings(tables, threads):
    engines, phys = tables
    for e in ne.int_expr_inputs():
        check(engines[threads], phys, "enc", None, ne.KEYS, ne._all4(e))
    if threads == 1:  # a NULL int64 key groups with 0; the key the oracle prints for that group follows its merge order
        check(engines[threads], phys, "enc", None, [ne.V], [lp.Count(lp.Col(ne.V)), lp.Sum(lp.Col(ne.T))])


@pytest.mark.parametrize("threads", [1, 4])
def test_float_aggregate_inputs(tables, threads):
    engines, phys = tables
    for aggs in ne.float_expr_aggs():
        if threads == 4 and float_nan_minmax(aggs):
            continue
        check(engines[threads], phys, "expr", None, ne.KEYS, aggs)


@pytest.mark.parametrize("threads", [1, 4])
def test_computed_keys(tables, threads):
    engines, phys = tables
    aggs = [lp.Sum(lp.Col(ne.V)), lp.Min(lp.Col(ne.V)), lp.Count(lp.Col(ne.V))]
    for keys in ne.computed_key_sets():
        check(engines[threads], phys, "expr", None, keys, aggs)


@pytest.mark.parametrize("threads", [1, 4])
def test_int64_and_packed_dictionary_keys(tables, threads):
    engines, phys = tables
    aggs = [lp.Sum(lp.Col(ne.T)), lp.Min(lp.Col(ne.T)), lp.Max(lp.Col(ne.T)), lp.Count(lp.Col(ne.T))]
    for keys in ([ne.V], [ne.V, "labels.a"], ["labels.b", ne.V, ne.bucket(7)]):
        check(engines[threads], phys, "ikeys", None, keys, aggs)
    for keys in ne.HASH_KEY_SETS:
        check(engines[threads], phys, "hkeys", None, keys, aggs)


def test_datasets_hold_what_the_cases_are_about(tables):
    _, phys = tables
    e = phys["expr"]
    assert min(e[0]["timestamp"]) < -1000 and max(e[0]["timestamp"]) > 1000
    ts = set(e[1]["timestamp"].tolist())
    assert set(ne.DIVISORS) <= ts
    assert ne.I64_MIN in set(e[1]["value"].tolist()) and ne.I64_MAX in set(e[1]["value"].tolist())
    assert all("floatvalue#valid" in p for p in e)
    # INT64_MIN / -1 happens, and wraps
    v, t = e[1]["value"], e[1]["timestamp"]
    assert ((v == ne.I64_MIN) & (t == -1)).any()
    assert ne.eval_expr(lp.Div(lp.Col(ne.V), lp.Literal(-1)), {"value": [ne.I64_MIN], "timestamp": [0]}).tolist() == [ne.I64_MIN]
    assert ne.eval_expr(lp.Div(lp.Col(ne.T), lp.Literal(1000)), {"timestamp": [-999, -1000, 999]}).tolist() == [0, -1, 0]
    for p in phys["enc"]:
        assert "value#valid" in p and (p["value"] == 0).any()
    k = phys["hkeys"][0]
    for name, card in (("labels.c", 4095), ("labels.d", 4096), ("labels.e", 9000)):
        assert None in set(k[name].tolist()) and f"v{card - 1:06d}" in set(k[name].tolist())


def test_written_encodings(tables):
    """The encoded parts are what they say: `value` as an optional PLAIN chunk with NULLs, and as CK_DICT64."""
    from frostdb_b200 import _lib
    for name, cols, buf in ne.encoded_parts(61):
        d = _lib.describe_parquet(buf)
        for rg in d["row_groups"]:
            c = rg["columns"]["value"]
            assert "error" not in c, c
            assert c["kind"] == (3 if name == "dict64" else 1), (name, c["kind"])
            assert c["n_values"] < rg["n_rows"], name
