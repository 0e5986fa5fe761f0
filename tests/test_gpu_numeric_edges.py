"""Numeric edges on every scan path against the plain reference of tests/numeric_edges.py (and, where the oracle's
NaN handling does not depend on its merge order, against the oracle too): int64 literals at the ends of the domain
on narrowed and 64-bit chunks, fused ranges that end up full, empty or one value wide, int columns against float
literals, IEEE specials in float columns, int64 sums that wrap, and the bound under which the tile kernel sums in
32-bit shared-memory cells without carries.

Each aggregate plan runs under every switch set of AGG_SWITCHES (sorted-run kernel k_runs_tma, tile kernel k_tile_agg
with and without its carry path and with its global table, fast_pass, the general k_scan, no pruning, no fusing);
filter-only plans run on the ordered take kernels and on k_rows.  With the default switches every aggregate case
asserts, from the result statistics, which kernel took its row groups."""
import ctypes as C
import os

import numpy as np
import pytest

from frostdb_b200 import _lib
from frostdb_b200 import dynparquet as dp
from frostdb_b200 import logicalplan as lp
from frostdb_b200 import query
from frostdb_b200.physicalplan import GPUScan
from tests import numeric_edges as ne
from tests.test_gpu_parity import Pair
from tests.util import label_values

pytestmark = pytest.mark.gpu

AGG_SWITCHES = [{}, {"FROSTGPU_NO_RUNS": "1"}, {"FROSTGPU_NO_RUNS": "1", "FROSTGPU_NO_TILE": "1"},
                {"FROSTGPU_NO_RUNS": "1", "FROSTGPU_NO_TILE": "1", "FROSTGPU_NO_FAST": "1"}, {"FROSTGPU_NO_PRUNE": "1"},
                {"FROSTGPU_NO_FUSE": "1"}, {"FROSTGPU_TA_GLOBAL": "1"}, {"FROSTGPU_TA_CARRY": "1"}]
ALL_SWITCHES = ("FROSTGPU_NO_RUNS", "FROSTGPU_NO_TILE", "FROSTGPU_NO_FAST", "FROSTGPU_NO_PRUNE", "FROSTGPU_NO_FUSE",
                "FROSTGPU_NO_TAKE", "FROSTGPU_TA_GLOBAL", "FROSTGPU_TA_CARRY", "FROSTGPU_TA_CHUNK", "FROSTGPU_TA_TILE")
N_ROWS = 2 * ne.RG * len(ne.INT_CHUNKS)
N_RG = len(ne.INT_CHUNKS)  # row groups per part
AGG_SC = [lp.Sum(lp.Col(ne.V)), lp.Count(lp.Col(ne.V))]  # one stored aggregate: fast_pass takes it


@pytest.fixture(autouse=True)
def clean_switches():
    yield
    for k in ALL_SWITCHES:
        os.environ.pop(k, None)


@pytest.fixture(scope="module")
def edges(store):
    """Two tables with the same sorted and unsorted part: with and without chunk statistics."""
    parts = [ne.int_part(ne.INT_CHUNKS, 11, sort=True), ne.int_part(ne.INT_CHUNKS, 12, sort=False, t0=N_ROWS // 2, part=1)]
    pairs = {}
    for stats in (True, False):
        p = Pair(store, f"numeric_edges_{int(stats)}", dp.SampleDefinitionWithFloat())
        for cols, sort in zip(parts, (True, False)):
            buf = ne.write(cols, sort=sort, stats=stats)
            p.gt.InsertParquet(buf)
            p.ot.InsertParquet(buf)
        pairs[stats] = p
    yield pairs, [ne.physical(c) for c in parts]
    for p in pairs.values():
        p.close()


def scan(q, filt):
    return q.Filter(filt) if filt is not None else q


def gpu_agg(p, filt, keys, aggs):
    out = []
    scan(query.NewEngine(None, p.db.TableProvider()).ScanTable(p.name), filt).Aggregate(aggs, [lp.Col(k) for k in keys]) \
        .Execute(None, lambda c, r: out.append(r))
    return ne.result_map(out, keys, aggs)


def oracle_agg(p, filt, keys, aggs):
    from tests.oracle_scan import oracle_query
    out = []
    scan(oracle_query(p.oe, p.name), filt).Aggregate(aggs, [lp.Col(k) for k in keys]).Execute(None, lambda c, r: out.append(r))
    return ne.result_map(out, keys, aggs)


def stats_of(store, name, filt, keys, aggs):
    eng, lib = store.engine, _lib.load()
    q, keep = GPUScan(eng, name, filt, _lib.PLAN_AGGREGATE, [lp.Col(k) for k in keys], aggs).prepare()
    res = C.c_void_p()
    try:
        _lib.check(lib.fgpu_query_execute(eng.handle, q, eng.table_watermark(name), C.byref(res)))
        st = eng.stats(res)
        lib.fgpu_result_free(res)
    finally:
        lib.fgpu_query_free(q)
    return st


def leaves(f):
    if f is None:
        return []
    if f.Op in (lp.OpAnd, lp.OpOr):
        return leaves(f.Left) + leaves(f.Right)
    return [f]


def runs_eligible(filt):
    """k_runs_tma takes plain int64 range leaves only: no `!=`, no float literal, no float column."""
    return all(l.Op != lp.OpNotEq and not isinstance(l.Right.Value, float) and l.Left.Name() != ne.F for l in leaves(filt))


def check_agg(p, phys, filt, aggs, keys=ne.KEYS, *, kernel=None, with_oracle=True, switches=AGG_SWITCHES):
    """Every switch set against the reference (and the oracle); with the default switches, `kernel(stats)` asserts the
    kernel that took the row groups."""
    what = f"{p.name} filter {filt.Name() if filt is not None else None} {[a.Name() for a in aggs]}"
    exp = ne.reference(phys, filt, keys, aggs)
    if with_oracle and not ne.has_nan_minmax(aggs):
        ne.assert_same_result(oracle_agg(p, filt, keys, aggs), exp, aggs, what + " oracle")
    for sw in switches:
        os.environ.update(sw)
        try:
            got = gpu_agg(p, filt, keys, aggs)
        finally:
            for k in sw:
                os.environ.pop(k)
        ne.assert_same_result(got, exp, aggs, f"{what} {sw}")
    if kernel is not None:
        st = stats_of(p.store, p.name, filt, keys, aggs)
        assert kernel(st), f"{what}: row groups {st['row_groups']}, runs {st['row_groups_runs']}, tiles {st['row_groups_tiles']}"


def edge_kernel(stats, filt):
    """Sorted row groups on k_runs_tma when the plan qualifies, every other row group on k_tile_agg.  Without
    statistics nothing is pruned, so the counts are exact."""
    runs = runs_eligible(filt)

    def ok(st):
        if stats:
            return st["row_groups_runs"] + st["row_groups_tiles"] == st["row_groups"] and (runs or st["row_groups_runs"] == 0)
        return st["row_groups"] == 2 * N_RG and st["row_groups_runs"] == (N_RG if runs else 0) and \
            st["row_groups_tiles"] == (N_RG if runs else 2 * N_RG)
    return ok


def check_take(p, phys, filt, names):
    exp = ne.reference_rows(phys, filt, names)
    for sw in ({}, {"FROSTGPU_NO_TAKE": "1"}):
        os.environ.update(sw)
        try:
            out = []
            query.NewEngine(None, p.db.TableProvider()).ScanTable(p.name).Filter(filt).Project(*[lp.Col(n) for n in names]) \
                .Execute(None, lambda c, r: out.append(r))
        finally:
            for k in sw:
                os.environ.pop(k)
        ne.assert_same_rows(ne.record_rows(out, names), exp, f"{p.name} {filt.Name()} {sw}")


@pytest.mark.parametrize("stats", [True, False])
def test_int64_literal_edges(edges, stats):
    pairs, phys = edges
    p = pairs[stats]
    for f in ne.int_edge_filters(N_ROWS):
        check_agg(p, phys, f, ne.AGG_INT, kernel=edge_kernel(stats, f))
        check_agg(p, phys, f, AGG_SC, with_oracle=False)


@pytest.mark.parametrize("stats", [True, False])
def test_int64_literal_edges_filter_only(edges, stats):
    pairs, phys = edges
    for f in ne.int_edge_filters(N_ROWS):
        check_take(pairs[stats], phys, f, [ne.T, ne.V])


@pytest.mark.parametrize("stats", [True, False])
def test_fused_conjunctions(edges, stats):
    pairs, phys = edges
    p = pairs[stats]
    for f in ne.fused_filters():
        check_agg(p, phys, f, ne.AGG_INT, kernel=edge_kernel(stats, f))
        check_agg(p, phys, f, AGG_SC, with_oracle=False)
        check_take(p, phys, f, [ne.T, ne.V, ne.F])


@pytest.mark.parametrize("stats", [True, False])
def test_int_column_against_float_literals(edges, stats):
    pairs, phys = edges
    p = pairs[stats]
    for f in ne.int_float_filters():
        check_agg(p, phys, f, ne.AGG_INT, kernel=edge_kernel(stats, f))
        check_take(p, phys, f, [ne.T, ne.V])


@pytest.mark.parametrize("stats", [True, False])
def test_float_specials(edges, stats):
    pairs, phys = edges
    p = pairs[stats]
    for f in [None] + ne.float_filters():
        check_agg(p, phys, f, ne.AGG_FLOAT, kernel=edge_kernel(stats, f))
        check_agg(p, phys, f, ne.AGG_FLOAT_SUM + [lp.Min(lp.Col(ne.V))])
    check_take(p, phys, ne.leaf(ne.F, lp.OpNotEq, ne.NAN), [ne.T, ne.F])
    check_take(p, phys, ne.leaf(ne.F, lp.OpGtEq, -ne.INF), [ne.T, ne.F])


@pytest.fixture(scope="module")
def wrapping(store):
    """Unsorted parts whose group sums cross +-2^63 many times: a dense table and one whose key dictionaries make the
    group space too large for it (hash-table mode)."""
    made = {}
    for name, kw in (("dense", {}), ("hash", {"ka": 3000, "kb": 2000, "used": (5, 7)})):
        p = Pair(store, f"numeric_wrap_{name}", dp.SampleDefinition())
        parts = [ne.wrap_part(50_000, 21, **kw), ne.wrap_part(30_000, 22, t0=50_000, **kw)]
        for cols in parts:
            p.insert(cols, sort=False, row_group_size=20_000)
        made[name] = (p, [ne.physical(c) for c in parts])
    yield made
    for p, _ in made.values():
        p.close()


def test_wrapping_sums_on_every_aggregate_kernel(wrapping):
    p, phys = wrapping["dense"]
    tiles = lambda st: st["row_groups_tiles"] == st["row_groups"] > 0  # noqa: E731
    general = lambda st: st["row_groups_tiles"] == st["row_groups_runs"] == 0 and st["row_groups"] > 0  # noqa: E731
    for aggs in (ne.AGG_INT, AGG_SC, [lp.Sum(lp.Col(ne.V)), lp.Max(lp.Col(ne.V))]):
        check_agg(p, phys, None, aggs, kernel=tiles)
        check_agg(p, phys, ne.leaf(ne.T, lp.OpGtEq, 7), aggs, kernel=tiles)
        check_agg(p, phys, lp.And(ne.leaf("labels.a", lp.OpNotEq, "v000001"), ne.leaf(ne.T, lp.OpLt, 70_000)), aggs, kernel=tiles)
        check_agg(p, phys, lp.Or(ne.leaf(ne.V, lp.OpLt, 0), ne.leaf(ne.T, lp.OpGt, 60_000)), aggs, kernel=general)
    p, phys = wrapping["hash"]
    for aggs in (ne.AGG_INT, AGG_SC):
        check_agg(p, phys, None, aggs, kernel=general)
        check_agg(p, phys, ne.leaf(ne.V, lp.OpGt, ne.I64_MIN), aggs, kernel=general)


# ---- the bound of the 32-bit shared-memory Sum (tile kernel, NOCARRY instance) ------------------------------------
NOCARRY_ROWS = 4 << 20


@pytest.mark.parametrize("value", [87_000, 93_300])  # under the host's bound with the default chunk; above it
@pytest.mark.parametrize("stats", [True, False])
def test_nocarry_bound(store, value, stats):
    """Sum(value) of a constant over 4 Mi unsorted rows by a one-value key (32 replicated shared-memory cells) and by
    two keys.  With a chunk override of 100000 tiles one CTA takes every tile, and each cell sees ~131 k rows: its
    32-bit sum must carry.  Expected: count * value, as Python ints."""
    rng = np.random.default_rng(value)
    n = NOCARRY_ROWS
    b = rng.integers(0, 3, n).astype(np.int32)
    cols = {
        "example_type": (np.zeros(n, np.int32), ["cpu"]),
        "stacktrace": (np.zeros(n, np.int32), ["s"]),
        "timestamp": np.arange(n, dtype=np.int64),
        "value": np.full(n, value, np.int64),
        "labels.a": (np.zeros(n, np.int32), label_values(1)),
        "labels.b": (b, label_values(3)),
    }
    name = f"numeric_nocarry_{value}_{int(stats)}"
    db = store.DB(None, "parity")
    if name in db.tables:
        store.engine.drop_table(name)
        db.tables.pop(name)
    t = db.Table(name, dp.SampleDefinition())
    t.InsertParquet(dp.write_part(dp.SampleDefinition(), cols, sort=False, row_group_size=1 << 20, write_statistics=stats))
    counts_b = np.bincount(b, minlength=3)
    try:
        for keys, exp in ((["labels.a"], {("v000000",): (n * value, n)}),
                          (["labels.a", "labels.b"], {("v000000", label_values(3)[i]): (int(counts_b[i]) * value, int(counts_b[i])) for i in range(3)})):
            for sw in ({}, {"FROSTGPU_TA_CHUNK": "100000"}, {"FROSTGPU_TA_CHUNK": "2"}, {"FROSTGPU_TA_CARRY": "1"}):
                sw = dict(sw, FROSTGPU_NO_RUNS="1")  # a constant key is one run: keep the row groups on the tile kernel
                os.environ.update(sw)
                try:
                    out = []
                    query.NewEngine(None, db.TableProvider()).ScanTable(name).Aggregate(AGG_SC, [lp.Col(k) for k in keys]) \
                        .Execute(None, lambda c, r: out.append(r))
                finally:
                    for k in sw:
                        os.environ.pop(k)
                got = ne.result_map(out, keys, AGG_SC)
                if got != exp:
                    wrong = {k: (v[0] - exp[k][0]) % (1 << 32) if k in exp else None for k, v in got.items()}
                    raise AssertionError(f"{keys} {sw}: got {got}, expected {exp} (difference mod 2^32: {wrong})")
        os.environ["FROSTGPU_NO_RUNS"] = "1"
        st = stats_of(store, name, None, ["labels.a"], AGG_SC)
        assert st["row_groups_tiles"] == st["row_groups"] == 4
    finally:
        store.engine.drop_table(name)
        db.tables.pop(name, None)


@pytest.mark.parametrize("tile", [6144, 3072])
def test_nocarry_bound_at_the_heaviest_cta(store, tile):
    """The host's bound itself, on one unreplicated shared-memory cell: 2048 key labels (a table too large for
    replicas), every row on the first one, (3 x SMs + 1) x 6144 rows, so the first CTA takes one tile more than the
    others.  `fits`: the largest value the bound allows without carries (max value x rows per CTA < 2^32); `wraps`: the
    smallest value whose 32-bit cell wraps in the heaviest CTA.  Both sums must be exact; a bound below the rows that
    CTA really takes would choose the carry-free instance for `wraps` and lose multiples of 2^32."""
    import torch
    G = torch.cuda.get_device_properties(0).multi_processor_count
    n = (3 * G + 1) * 6144
    t = n // tile
    chunk = max(1, t // (G * 4))
    assert chunk == 1
    heaviest = -(-t // G) * tile                       # tiles b, b + G, ...: the first CTA takes ceil(t / G)
    bound_rows = (t // G + 2 * chunk + 1) * tile       # the host's rows-per-CTA bound (engine.cpp, sums_fit32)
    fits, wraps = 0xFFFFFFFF // bound_rows, (1 << 32) // heaviest + 1
    assert wraps * bound_rows >= 1 << 32 and fits * heaviest < 1 << 32
    db = store.DB(None, "parity")
    for value in (fits, wraps):
        name = f"numeric_nocarry_cell_{tile}_{value}"
        if name in db.tables:
            store.engine.drop_table(name)
            db.tables.pop(name)
        cols = {
            "example_type": (np.zeros(n, np.int32), ["cpu"]),
            "stacktrace": (np.zeros(n, np.int32), ["s"]),
            "timestamp": np.arange(n, dtype=np.int64),
            "value": np.full(n, value, np.int64),
            "labels.a": (np.zeros(n, np.int32), label_values(2048)),
        }
        t_ = db.Table(name, dp.SampleDefinition())
        t_.InsertParquet(dp.write_part(dp.SampleDefinition(), cols, sort=False, row_group_size=64 * 6144))
        sw = {"FROSTGPU_NO_RUNS": "1", "FROSTGPU_TA_TILE": str(tile)}  # a constant key is one run: keep the tile kernel
        os.environ.update(sw)
        try:
            out = []
            query.NewEngine(None, db.TableProvider()).ScanTable(name).Aggregate(AGG_SC, [lp.Col("labels.a")]) \
                .Execute(None, lambda c, r: out.append(r))
            got = ne.result_map(out, ["labels.a"], AGG_SC)
            exp = {("v000000",): (n * value, n)}
            assert got == exp, f"tile {tile} value {value}: got {got}, expected {exp}"
            st = stats_of(store, name, None, ["labels.a"], AGG_SC)
            assert st["row_groups_tiles"] == st["row_groups"] > 0
        finally:
            for k in sw:
                os.environ.pop(k)
            store.engine.drop_table(name)
            db.tables.pop(name, None)


# ---- the known divergence from Go: NaN as the first value of a group ------------------------------------------------
@pytest.mark.xfail(strict=True, reason="Go's Min / Max keep a NaN that comes first in a group (and return NaN for a group of "
                                       "NaNs); the kernels never select NaN and return the other values' extreme or the "
                                       "reducer's identity (DESIGN §2, unpinned)")
def test_nan_first_in_group_min_max(store):
    p = Pair(store, "numeric_nan_first", dp.SampleDefinitionWithFloat())
    try:
        n = 64
        cols = {
            "example_type": (np.zeros(n, np.int32), ["cpu"]),
            "stacktrace": (np.zeros(n, np.int32), ["s"]),
            "timestamp": np.arange(n, dtype=np.int64),
            "value": np.arange(n, dtype=np.int64),
            "labels.a": (np.repeat(np.arange(2, dtype=np.int32), n // 2), label_values(2)),
            "floatvalue": np.r_[[ne.NAN], np.arange(1, n // 2, dtype=np.float64), np.full(n // 2, ne.NAN)],
        }
        p.insert(cols, sort=False)
        aggs = [lp.Min(lp.Col(ne.F)), lp.Max(lp.Col(ne.F))]
        exp = ne.reference([ne.physical(cols)], None, ["labels.a"], aggs)
        assert all(v != v for vals in exp.values() for v in vals)  # Go's answer: NaN for both groups
        ne.assert_same_result(gpu_agg(p, None, ["labels.a"], aggs), exp, aggs, "NaN first")
    finally:
        p.close()
