"""Every reachable instance of the specialised scan kernels (tests/kernel_instances.py) against the exact reference of
tests/numeric_edges.py: Sum(int64) wraps modulo 2^64, float Sums are order independent (integer-valued), Min / Max at
the ends of int64, filter-only rows in order.

One table per kernel family, built once, with its data placed where that family's instances differ:
- `runs`: sorted parts with labels.a / .b / .c in long runs (run-length-only chunks) and, in one row group per part, a
  stretch of 16-row runs that overflows the staged directory window.  Row group 0 of every part passes both range
  leaves whole, row group 1 is pruned, row groups 2 and 3 are filtered row by row; their int64 columns stage at 1, 2,
  4 and 8 bytes, at the ends of int64.  Every case runs under four switch sets.
- `tiles`: unsorted parts, four nullable keys with 8-bit codes, one with 16-bit and one with a 70 000-value dictionary
  (a dense table over 227 KB), one part without labels.d; bounded (`u`, `x`) and wide (`value`, `timestamp`) Sum inputs.
- `take`: a permutation in `value` (every selectivity without pruning), 1 to 4 projected PLAIN columns.
- `prefix`: sorted row groups whose labels.c slots collect >= 256 segments each, and keys with few segments per slot.
- `fast`: parts holding 3, 2, 1 and 0 of the plan's keys; row groups leaving 2, 1 and 0 leaves undecided.

The last test prints which tuples ran under which switches and which are unreachable, and fails when a reachable tuple
did not run."""
import ctypes as C
import os

import numpy as np
import pytest

from frostdb_b200 import _lib
from frostdb_b200 import dynparquet as dp
from frostdb_b200 import logicalplan as lp
from frostdb_b200.physicalplan import GPUScan
from tests import kernel_instances as ki
from tests import numeric_edges as ne
from tests.util import label_values

pytestmark = pytest.mark.gpu

I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
V, T, W, X, U, F = ki.V, ki.T, ki.W, ki.X, ki.U, ki.F
SCHEMA = dp.Schema("kinst", [dp.ColumnDefinition("labels", dp.TYPE_STRING, nullable=True, dynamic=True, rle_dictionary=True)]
                   + [dp.ColumnDefinition(c, dp.TYPE_INT64) for c in ki.INT_COLS] + [dp.ColumnDefinition(F, dp.TYPE_DOUBLE)],
                   [dp.SortingColumn("labels", nulls_first=True), dp.SortingColumn("timestamp")])
COVER = {k: {} for k in ki.KERNELS}  # kernel -> instance -> {switch label: what ran}


def label_of(env) -> str:
    return ",".join(f"{k}={v}" for k, v in sorted(dict(env).items())) or "default"


def values(rng, lo: int, hi: int, n: int) -> np.ndarray:
    """n int64 values in [lo, hi], both ends present."""
    v = [lo + int(x) % (hi - lo + 1) for x in rng.integers(0, 1 << 62, n, dtype=np.int64)]
    v[int(rng.integers(0, n))], v[int(rng.integers(0, n))] = lo, hi
    return np.array(v, dtype=np.int64)


def int_floats(rng, lo: int, hi: int, n: int) -> np.ndarray:
    """Integer-valued doubles: every Sum is exact in any order."""
    return values(rng, lo, hi, n).astype(np.float64)


def put(store, name, parts):
    """A table of `parts` (column dicts, written in the order given) -> (name, the reference's view of every part)."""
    eng = store.engine
    eng.drop_table(name)
    for cols, rg in parts:
        eng.put_parquet(name, dp.write_part(SCHEMA, cols, sort=False, row_group_size=rg))
    names = set().union(*[cols for cols, _ in parts])
    phys = []
    for cols, _ in parts:
        p = ne.physical(cols)
        n = len(p[T])
        for c in names - set(cols):  # a column the part does not have: NULL in every row
            p[c] = np.full(n, None, dtype=object)
        phys.append(p)
    return name, phys


# ---- tables -----------------------------------------------------------------------------------------------------------
RUNS_RG = 8192
# per part, per row group: (lo, hi) of value, timestamp, w, x.  Leaves `value >= 0`, `timestamp <= 100`: row group 0
# passes both, row group 1 fails the first, row groups 2 and 3 are cut by one and pass the other.
RUNS_RANGES = [
    [((1000, 1255), (-65536, -1), (-7, 248), (1000, 1256)),
     ((-(1 << 40), -(1 << 40) + 255), (0, 65535), (3, 65539), (-(1 << 31), (1 << 31) - 1)),
     ((I64_MIN, I64_MAX), (-7, 248), (I64_MIN, I64_MAX), (I64_MIN, I64_MIN + 70_000)),
     ((-(1 << 31), (1 << 31) - 1), (I64_MIN, I64_MIN + 65535), (I64_MAX - 200, I64_MAX), (-1, 0))],
    [((I64_MAX - 200, I64_MAX), (I64_MIN, I64_MIN + (1 << 32) - 1), (17, 17 + (1 << 32)), (I64_MAX - (1 << 32) + 1, I64_MAX)),
     ((I64_MIN, I64_MIN + 70_000), (0, 100), (-1, 0), (-7, 248)),
     ((-1, 0), (-(1 << 31), (1 << 31) - 1), (I64_MIN, I64_MIN + 65535), (I64_MIN, I64_MAX)),
     ((I64_MIN, I64_MAX), (-(1 << 40), -(1 << 40) + 65535), (1000, 1255), (3, 65539))],
]
RUNS_SHORT_RG = (2, 3)  # the row group of each part that starts with 2048 rows of 16-row runs


def runs_part(seed, ranges, short_rg):
    rng = np.random.default_rng(seed)
    n = RUNS_RG * len(ranges)
    seg = np.empty(n, np.int64)
    r, sid = 0, int(rng.integers(0, 60))
    while r < n:  # run lengths are multiples of 8: every run is an RLE run of the dictionary indices
        short = short_rg * RUNS_RG <= r < short_rg * RUNS_RG + 2048
        ln = 16 if short else int(rng.choice([128, 192, 256, 384]))
        seg[r:r + ln] = sid
        r, sid = r + ln, sid + 1
    seg = seg[:n]
    cols = {"labels.a": (((seg // 20) % 3).astype(np.int32), label_values(3)),
            "labels.b": (((seg // 5) % 4).astype(np.int32), label_values(4)),
            "labels.c": ((seg % 5).astype(np.int32), label_values(5)),
            F: int_floats(rng, -(1 << 20), 1 << 20, n)}
    for i, c in enumerate((V, T, W, X)):
        cols[c] = np.concatenate([values(rng, *rr[i], RUNS_RG) for rr in ranges])
    return cols


TILE_ROWS = ki.TILE_RG * ki.TILE_RGS_PER_PART


def tile_part(seed, part):
    rng = np.random.default_rng(seed)
    n = TILE_ROWS
    cols = {}
    for k, card in ki.TILE_CARD.items():
        if (k, part) == ki.TILE_ABSENT_KEY:
            continue
        idx = rng.integers(0, card, n).astype(np.int32)
        idx[rng.random(n) < 0.05] = -1
        idx[int(rng.integers(0, n))] = card - 1
        cols[k] = (idx, label_values(card))
    cols[V] = values(rng, I64_MIN, I64_MAX, n)
    cols[T] = values(rng, -(1 << 62), 1 << 62, n)
    cols[U] = values(rng, 0, ki.U_MAX, n)
    cols[X] = values(rng, 0, ki.U_MAX, n)
    cols[F] = int_floats(rng, -(1 << 30), 1 << 30, n)
    return cols


def take_part(seed):
    rng = np.random.default_rng(seed)
    n = ki.TAKE_ROWS
    v = np.arange(n + 1, dtype=np.int64)
    v = rng.permutation(v[v != ki.TAKE_ABSENT])
    return {V: v, T: np.arange(n, dtype=np.int64), W: values(rng, I64_MIN, I64_MAX, n), F: int_floats(rng, -(1 << 40), 1 << 40, n),
            "labels.a": (rng.integers(0, 3, n).astype(np.int32), label_values(3)),
            "labels.b": (rng.integers(0, 2, n).astype(np.int32), label_values(2))}


def prefix_part(seed):
    rng = np.random.default_rng(seed)
    rg, n = ki.PREFIX_RG, ki.PREFIX_RG * ki.PREFIX_RGS
    row = np.arange(n) % rg
    runs = ki.PREFIX_RUNS
    cols = {k: (((row // (rg // runs[k])) % ki.PREFIX_CARD[k]).astype(np.int32), label_values(ki.PREFIX_CARD[k])) for k in runs}
    cols[V] = values(rng, I64_MIN, I64_MAX, n)
    cols[T] = values(rng, -(1 << 62), 1 << 62, n)
    return cols


# per row group r of every part: value and timestamp leave 2 - r of the leaves `x >= 0`, `timestamp >= 0` undecided
FAST_RANGES = [((-500, 500), (-100, 100)), ((-500, 500), (0, 1000)), ((0, 1000), (0, 1000))]


def fast_part(seed, part):
    rng = np.random.default_rng(seed)
    rg = ki.FAST_RG
    n = rg * ki.FAST_RGS_PER_PART
    cols = {k: (rng.integers(0, card, n).astype(np.int32), label_values(card))
            for k, card in zip(ki.FAST_KEYS_ALL[:ki.FAST_KEYS - part], (3, 4, 5))}
    cols[V] = np.concatenate([values(rng, *r[0], rg) for r in FAST_RANGES])
    cols[T] = np.concatenate([values(rng, *r[1], rg) for r in FAST_RANGES])
    cols[F] = np.concatenate([int_floats(rng, *r[0], rg) for r in FAST_RANGES])
    return cols


@pytest.fixture(scope="module")
def tables(store):
    made = {
        "runs": put(store, "kinst_runs", [(runs_part(7100 + p, rr, RUNS_SHORT_RG[p]), RUNS_RG) for p, rr in enumerate(RUNS_RANGES)]),
        "tiles": put(store, "kinst_tiles", [(tile_part(7200 + p, p), ki.TILE_RG) for p in range(ki.TILE_PARTS)]),
        "take": put(store, "kinst_take", [(take_part(7300), ki.TAKE_RG)]),
        "prefix": put(store, "kinst_prefix", [(prefix_part(7400), ki.PREFIX_RG)]),
        "fast": put(store, "kinst_fast", [(fast_part(7500 + p, p), ki.FAST_RG) for p in range(ki.FAST_PARTS)]),
    }
    yield made
    for name, _ in made.values():
        store.engine.drop_table(name)


def execute(store, table, s: ki.Shape, env):
    """One prepared plan under the switches `env`, executed once: (records, stats)."""
    eng, lib = store.engine, _lib.load()
    rows_plan = bool(s.out)
    os.environ.update(dict(env))
    try:
        scan = GPUScan(eng, table, s.filter, _lib.PLAN_FILTER if rows_plan else _lib.PLAN_AGGREGATE,
                       [lp.Col(c) for c in (s.out if rows_plan else s.keys)], [] if rows_plan else list(s.aggs))
        q, keep = scan.prepare()
        res = C.c_void_p()
        try:
            _lib.check(lib.fgpu_query_execute(eng.handle, q, eng.table_watermark(table), C.byref(res)))
            try:
                recs = list(eng.drain(res))
                st = eng.stats(res)
            finally:
                lib.fgpu_result_free(res)
        finally:
            lib.fgpu_query_free(q)
    finally:
        for k in dict(env):
            os.environ.pop(k, None)
    return recs, st


def check_aggregate(store, tables, s: ki.Shape, env, exp=None):
    table, parts = tables[s.table]
    if exp is None:
        exp = ne.reference(parts, s.filter, list(s.keys), list(s.aggs))
    recs, st = execute(store, table, s, env)
    ne.assert_same_result(ne.result_map(recs, list(s.keys), list(s.aggs)), exp, list(s.aggs), f"{s.name()} under {label_of(env)}")
    return exp, st


def ids(shapes):
    return [f"{s.instance}-{s.note or i}".replace(" ", "") for i, s in enumerate(shapes)]


# ---- k_runs_tma ---------------------------------------------------------------------------------------------------------
RUNS = ki.shapes("k_runs_tma")


@pytest.mark.parametrize("s", RUNS, ids=ids(RUNS))
def test_runs_tma_instance(store, tables, s):
    exp = None
    nl = s.instance[0]
    for env in ki.RUNS_SWITCHES:
        exp, st = check_aggregate(store, tables, s, env, exp)
        assert st["row_groups_runs"] == st["row_groups"], (s.name(), env, st)
        assert st["row_groups_pruned"] == (2 if nl else 0), (s.name(), env, st)
        tma = st["row_groups_runs"] - st["row_groups_prefix"]
        # without range leaves every row group is all-pass: Sum-only plans without undecided dictionary leaves may be
        # answered from prefix sums alone
        assert tma > 0 or st["row_groups_prefix"] == st["row_groups"], (s.name(), env, st)
        COVER["k_runs_tma"].setdefault(s.instance, {})[label_of(env)] = "k_runs_tma" if tma else "prefix sums only"


# ---- k_tile_agg --------------------------------------------------------------------------------------------------------
TILES = ki.shapes("k_tile_agg")


@pytest.mark.parametrize("s", TILES, ids=ids(TILES))
def test_tile_agg_instance(store, tables, s):
    _, st = check_aggregate(store, tables, s, s.env)
    assert st["row_groups_tiles"] == st["row_groups"] > 0, (s.name(), st)
    COVER["k_tile_agg"].setdefault(s.instance, {})[label_of(s.env)] = "k_tile_agg"


# ---- k_take_count / k_take_write ---------------------------------------------------------------------------------------
TAKES = ki.shapes("k_take_write")


@pytest.mark.parametrize("s", TAKES, ids=ids(TAKES))
def test_take_instances(store, tables, s):
    """The rows in order, on the take kernels (two more launches than k_rows under FROSTGPU_NO_TAKE)."""
    table, parts = tables[s.table]
    exp = ne.reference_rows(parts, s.filter, list(s.out))
    launches = {}
    for env in ({}, {"FROSTGPU_NO_TAKE": "1"}):
        recs, st = execute(store, table, s, env)
        ne.assert_same_rows(ne.record_rows(recs, list(s.out)), exp, f"{s.name()} ({s.note}) under {label_of(env)}")
        assert st["row_groups_pruned"] == 0, (s.name(), st)
        launches[label_of(env)] = st["kernel_launches"]
    assert launches["default"] == launches["FROSTGPU_NO_TAKE=1"] + 2, (s.name(), launches)
    COVER["k_take_write"].setdefault(s.instance, {})["default"] = f"k_take_write, {len(exp)} rows"
    COVER["k_take_count"].setdefault((s.instance[0], s.instance[2]), {})["default"] = "k_take_count"


# ---- k_runs_prefix -----------------------------------------------------------------------------------------------------
PREFIX = ki.shapes("k_runs_prefix")


@pytest.mark.parametrize("s", PREFIX, ids=ids(PREFIX))
def test_runs_prefix_instance(store, tables, s):
    exp, st = check_aggregate(store, tables, s, {})
    assert st["row_groups_prefix"] == st["row_groups"] == ki.PREFIX_RGS, (s.name(), st)
    check_aggregate(store, tables, s, {"FROSTGPU_NO_PREFIX": "1"}, exp)
    COVER["k_runs_prefix"].setdefault(s.instance, {})["default"] = f"{ki.prefix_segments_per_slot(s)} segments per slot"


# ---- fast_pass / fast_pass_tight ---------------------------------------------------------------------------------------
FAST = {}
for _s in ki.shapes("fast_pass"):
    FAST.setdefault((_s.filter.Name(), tuple(a.Name() for a in _s.aggs)), []).append(_s)
FAST_PLANS = list(FAST.values())


@pytest.mark.parametrize("group", FAST_PLANS, ids=[",".join(a.Name() for a in g[0].aggs) + "|" + g[0].filter.Name() for g in FAST_PLANS])
def test_fast_pass_instances(store, tables, group):
    """One plan whose row groups select twelve (NL, NK) tuples of one (NA, tight)."""
    s = group[0]
    _, st = check_aggregate(store, tables, s, s.env)
    assert st["row_groups_runs"] == st["row_groups_tiles"] == 0 and st["row_groups"] == ki.FAST_PARTS * ki.FAST_RGS_PER_PART, st
    for g in group:
        COVER["fast_pass"].setdefault(g.instance, {})[label_of(g.env)] = f"row group {g.facts['row_group']}"


# ---- coverage ----------------------------------------------------------------------------------------------------------
def test_every_reachable_instance_ran():
    lines, missing = [], []
    for k in ki.KERNELS:
        reach = [t for t in ki.all_instances(k) if t not in ki.UNREACHABLE[k]]
        ran = COVER[k]
        lines.append(f"{k}: {sum(1 for t in reach if t in ran)} of {len(reach)} reachable tuples ran, {len(ki.UNREACHABLE[k])} unreachable")
        for t in reach:
            if t not in ran:
                missing.append((k, t))
            else:
                lines.append(f"  {t}: " + "; ".join(f"{e}: {w}" for e, w in sorted(ran[t].items())))
        for t, why in ki.UNREACHABLE[k].items():
            lines.append(f"  {t}: unreachable: {why}")
        if k == "k_runs_tma":
            for t in reach:
                if t in ran and len(ran[t]) != len(ki.RUNS_SWITCHES):
                    missing.append((k, t, "not under every switch set"))
                if t in ran and ran[t].get("FROSTGPU_NO_PREFIX=1") != "k_runs_tma":
                    missing.append((k, t, "k_runs_tma did not run with the prefix path off"))
    print("\n".join(lines))
    assert not missing, f"reachable tuples that did not run: {missing[:10]}"
