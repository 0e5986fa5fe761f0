"""Every compiled instance of the specialised scan kernels, and a plan shape that selects each one.

The hot path is a family of template instances; the host picks one from the plan's shape and from facts of the data
(code widths, chunk statistics, table size).  This module lists, for each kernel,

- every template-argument tuple the library compiles (`all_instances`), checked against the built library's symbols by
  tests/test_host_kernel_instances.py;
- a `Shape` per reachable tuple: filter leaves, group keys and aggregates as logicalplan expressions, the test table it
  runs on and the switches it runs under, run against the exact reference by tests/test_gpu_kernel_instances.py;
- the tuples no plan can select, each with the planner rule that rules it out (`UNREACHABLE`).

`expected_instance(kernel, shape)` restates each chooser in a few lines; it and the chooser it cites change together.
Pure Python: nothing here needs a GPU."""
from __future__ import annotations

import itertools
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

from frostdb_b200 import logicalplan as lp

KERNELS = ("k_runs_tma", "k_tile_agg", "k_take_count", "k_take_write", "k_runs_prefix", "fast_pass")

# limits the choosers clamp to (device_types.h, kernels.cu)
RUNS_LEAVES, RUNS_KEYS, RUNS_AGGS = 2, 3, 3            # kRunsLeaves, kRunsKeys, kRunsAggs
TA_KEYS, TA_SIMPLE_AGGS = 4, 2                         # kTaKeys; simple_smem_na has NA 0..2
TAKE_LEAVES, TAKE_OUT = 2, 4                           # kTakeLeaves, kTakeOut
FAST_LEAVES, FAST_KEYS, FAST_AGGS = 2, 3, 2            # kFastLeaves, kFastKeys, kFastAggs
PREFIX_CTA_SEGMENTS = 256                              # prefix_build: a CTA per slot from 256 segments per slot
TA_SMEM_MAX = 227 * 1024                               # tile_layout's kSmemMax

V, T, W, X, U, F = "value", "timestamp", "w", "x", "u", "floatvalue"
INT_COLS = (V, T, W, X, U)


def col(name: str) -> lp.Expr:
    return lp.Col(name)


def lit(v) -> lp.Expr:
    return lp.Literal(v)


def conj(leaves) -> Optional[lp.Expr]:
    leaves = list(leaves)
    if not leaves:
        return None
    return leaves[0] if len(leaves) == 1 else lp.And(*leaves)


# ---- the test tables: the facts the choosers read --------------------------------------------------------------------
# Sorted tables ("runs", "prefix"): dictionary keys in long runs.  Unsorted ("tiles", "fast"), and "take".
# Dictionary cardinalities (without NULL) of the key columns, and the code width of each in the tile table's flat
# code arrays: card + NULL <= 255 is 8 bits, <= 65535 16 bits, else 32 bits.
TILE_CARD = {"labels.a": 5, "labels.b": 3, "labels.c": 2, "labels.d": 2, "labels.w": 300, "labels.e": 70_000}
TILE_RG, TILE_PARTS, TILE_RGS_PER_PART = 6144, 3, 2
TILE_ABSENT_KEY = ("labels.d", 2)  # (column, part): the part that does not have the column
U_MAX = 100_000                    # `u` and `x` in the tile table: [0, U_MAX], statistics written (Sum fits 32 bits)
TILE_BOUNDED = {U, X}


def code_bits(card: int) -> int:
    n = card + 1  # NULL is code 0
    return 8 if n <= 255 else (16 if n <= 65535 else 32)


PREFIX_RG, PREFIX_RGS = 16_384, 4
PREFIX_MANY_RUNS = 256  # runs of labels.c per row group in the table whose key slots collect >= 256 segments


# ---- shapes -----------------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class Shape:
    """One plan: a conjunction of leaves, group keys (dictionary columns) and aggregates (or, for filter-only plans,
    projected columns), on `table`, under the switches `env`."""
    kernel: str
    instance: tuple
    table: str
    leaves: Tuple[lp.Expr, ...] = ()
    keys: Tuple[str, ...] = ()
    aggs: Tuple[lp.AggregationFunction, ...] = ()
    out: Tuple[str, ...] = ()  # filter-only plans: projected columns
    env: Tuple[Tuple[str, str], ...] = ()
    note: str = ""
    facts: Dict[str, object] = field(default_factory=dict, compare=False, hash=False)

    @property
    def filter(self):
        return conj(self.leaves)

    def name(self) -> str:
        f = self.filter
        what = ",".join(self.out) if self.out else ",".join(a.Name() for a in self.aggs)
        return f"{self.kernel}{self.instance} on {self.table}: {what} by {list(self.keys)} where {f.Name() if f is not None else None} {dict(self.env)}"


def _leaf_kind(e: lp.Expr) -> str:
    """'range': an int64 column against an int literal (<, <=, >, >=, ==); 'neg': != on an int64 column; 'float': a
    float64 column or a float literal; 'dict': a dictionary column."""
    name, v = e.Left.Name(), e.Right.Value
    if name.startswith("labels."):
        return "dict"
    if name == F or isinstance(v, float):
        return "float"
    return "neg" if e.Op == lp.OpNotEq else "range"


def _stored(aggs) -> list:
    return [a for a in aggs if a.Func != lp.AggFuncCount]


def _sum_int(a) -> bool:
    return a.Func == lp.AggFuncSum and a.Expr.Name() != F


# ---- the choosers, restated -------------------------------------------------------------------------------------------
def expected_instance(kernel: str, s: Shape) -> tuple:
    kinds = [_leaf_kind(e) for e in s.leaves]
    stored = _stored(s.aggs)
    if kernel == "k_runs_tma":
        # runs_query: range leaves / dictionary leaves / keys / Sum-Min-Max; pick -> pick_nl / pick_nk / pick_na
        nl, np_, nk, na = kinds.count("range"), kinds.count("dict"), len(s.keys), len(stored)
        gen = any(not _sum_int(a) for a in stored)
        return (min(nl, RUNS_LEAVES), min(nk, RUNS_KEYS), min(na, RUNS_AGGS), gen and na > 0, np_ > 0)
    if kernel == "k_tile_agg":
        # tile_query (leaf_flags, cell64), tile_layout (smem_table, keys8, sums_fit32), launch_tile_agg's `simple`
        # and simple_smem (NA 0..2 only)
        env = dict(s.env)
        simple = all(k == "range" for k in kinds) and all(_sum_int(a) for a in stored)
        nk, na = len(s.keys), len(stored)
        smem = "FROSTGPU_TA_GLOBAL" not in env and tile_table_bytes(s) + tile_min_ring(s) <= TA_SMEM_MAX
        k8 = all(code_bits(TILE_CARD[k]) <= 8 for k in s.keys)
        nocarry = "FROSTGPU_TA_CARRY" not in env and all(a.Expr.Name() in TILE_BOUNDED for a in stored)
        if simple and smem and na <= TA_SIMPLE_AGGS:
            return (True, True, nk, na, k8, nocarry)
        return (smem, simple, -1, -1, False, False)
    if kernel == "k_take_count":  # take_hp: NL 0..2, HP = any dictionary leaf
        return (min(kinds.count("range"), TAKE_LEAVES), kinds.count("dict") > 0)
    if kernel == "k_take_write":  # take_hp -> write_no
        return (min(kinds.count("range"), TAKE_LEAVES), min(len(s.out), TAKE_OUT), kinds.count("dict") > 0)
    if kernel == "k_runs_prefix":
        # prefix_build: group_log2 = 8 once ceil(seg_bound / n_slots) >= 256; launch_runs_prefix: kCta = group_log2 > 5
        return (prefix_segments_per_slot(s) >= PREFIX_CTA_SEGMENTS,)
    if kernel == "fast_pass":
        # build_fast_plan, per row group: leaves left undecided, keys present, stored aggregates; tight unless an
        # undecided leaf is not a plain int64 range or an aggregate is not Sum(int64)
        f = s.facts
        undecided = [k for k, d in zip(kinds, f["decided"]) if not d]
        tight = all(k == "range" for k in undecided) and all(_sum_int(a) for a in stored)
        return (len(undecided), f["keys_present"], len(stored), tight)
    raise KeyError(kernel)


def tile_table_bytes(s: Shape) -> int:
    """tile_layout: counts (4 bytes) + one cell per stored aggregate (4 bytes for an int64 Sum, else 8) per slot and
    replica; replicas while the table stays within 2048 cells."""
    slots = 1
    for k in s.keys:
        slots *= TILE_CARD[k] + 1
    rl = 0
    while rl < 5 and (slots << (rl + 1)) <= 2048:
        rl += 1
    cells = slots << rl
    tb = (cells * 4 + 7) & ~7
    for a in _stored(s.aggs):
        tb += (cells * (4 if _sum_int(a) else 8) + 7) & ~7
    return tb


def tile_min_ring(s: Shape) -> int:
    """The smallest ring tile_layout tries (768 rows, 2 stages) for the staged columns of the plan."""
    plain = {a.Expr.Name() for a in _stored(s.aggs)} | {e.Left.Name() for e in s.leaves if not e.Left.Name().startswith("labels.")}
    codes = set(s.keys) | {e.Left.Name() for e in s.leaves if e.Left.Name().startswith("labels.")}
    slot = len(plain) * 768 * 8 + sum((768 * max(code_bits(TILE_CARD.get(c, 1)), 8) // 8 + 127) & ~127 for c in codes)
    return 128 + 2 * (256 + max(slot, 128))


def prefix_window_rows(n_rows: int, sum_runs: int) -> int:
    """runs_prefix_window_rows."""
    if sum_runs == 0:
        return max(n_rows, 1)
    t = (32 * n_rows // sum_runs) & ~(128 - 1)  # kIndexRows = 128
    return min(max(t, 1024), max(n_rows, 1))


def prefix_segments_per_slot(s: Shape) -> int:
    """prefix_admit's segment bound (every key run start and every window start of every row group) over the dense
    slots, from the runs the prefix table is built with (facts: runs per key column per row group)."""
    runs, n_rows, n_rgs = s.facts["runs"], s.facts["rows"], s.facts["row_groups"]
    sum_runs = sum(runs[k] for k in s.keys)
    n_win = -(-n_rows // prefix_window_rows(n_rows, sum_runs))
    slots = 1
    for k in s.keys:
        slots *= s.facts["card"][k] + 1
    return -(-(n_rgs * (sum_runs + n_win)) // slots)


# ---- every compiled tuple, and the ones no plan selects ---------------------------------------------------------------
B = (False, True)


def all_instances(kernel: str) -> List[tuple]:
    if kernel == "k_runs_tma":
        na_gen = [(0, False)] + [(na, g) for g in B for na in (1, 2, 3)]
        return [(nl, nk, na, g, hp) for nl in range(3) for nk in range(4) for na, g in na_gen for hp in B]
    if kernel == "k_tile_agg":
        simple = [(True, True, nk, na, k8, nc) for nk in range(5) for na in range(3) for k8 in B for nc in B]
        return simple + [(sm, si, -1, -1, False, False) for sm in B for si in B]
    if kernel == "k_take_count":
        return [(nl, hp) for nl in range(3) for hp in B]
    if kernel == "k_take_write":
        return [(nl, no, hp) for nl in range(3) for no in range(1, 5) for hp in B]
    if kernel == "k_runs_prefix":
        return [(False,), (True,)]
    if kernel == "fast_pass":
        return [(nl, nk, na, t) for nl in range(FAST_LEAVES + 1) for nk in range(FAST_KEYS + 1) for na in range(FAST_AGGS + 1) for t in B]
    raise KeyError(kernel)


def _unreachable() -> Dict[str, Dict[tuple, str]]:
    out: Dict[str, Dict[tuple, str]] = {k: {} for k in KERNELS}
    for na, nc in itertools.product(range(3), B):
        out["k_tile_agg"][(True, True, 0, na, False, nc)] = \
            "tile_layout starts keys8 at 1 and clears it only for a key code column wider than 8 bits: a plan without keys is always K8"
    for nk in range(4):
        out["fast_pass"][(0, nk, 0, False)] = \
            "build_fast_plan clears `tight` only for an undecided non-plain leaf or a stored aggregate other than Sum(int64): no leaf and no stored aggregate is tight"
    return out


UNREACHABLE = _unreachable()


# ---- the shapes -------------------------------------------------------------------------------------------------------
RUNS_KEYS_ALL = ("labels.a", "labels.b", "labels.c")
# range leaves of the sorted table: in every part, row group 0 passes both whole, row group 1 fails `value >= 0`
# whole (pruned), row groups 2 and 3 are filtered row by row (see the table in test_gpu_kernel_instances.py)
RUNS_RANGE = (col(V).GtEq(lit(0)), col(T).LtEq(lit(100)))
RUNS_DICT = (col("labels.a").NotEq(lit("v000001")), col("labels.b").NotEq(lit("v000002")))
RUNS_AGG_SETS = {
    (0, False): (),
    (1, False): (lp.Sum(col(W)),),
    (2, False): (lp.Sum(col(W)), lp.Sum(col(X))),
    (3, False): (lp.Sum(col(W)), lp.Sum(col(X)), lp.Sum(col(V))),
    (1, True): (lp.Max(col(X)),),
    (2, True): (lp.Min(col(W)), lp.Sum(col(F))),
    # with both range leaves: five distinct staged columns, the fullest stage header
    (3, True): (lp.Min(col(W)), lp.Max(col(X)), lp.Sum(col(F))),
}
RUNS_SWITCHES = ({}, {"FROSTGPU_NO_PREFIX": "1"}, {"FROSTGPU_RT_WARPS": "4"}, {"FROSTGPU_RT_TILE": "1024"})


def runs_shapes() -> List[Shape]:
    out = []
    for nl, nk, hp in itertools.product(range(3), range(4), B):
        for (na, gen), aggs in RUNS_AGG_SETS.items():
            leaves = RUNS_RANGE[:nl] + (RUNS_DICT[:1 + nk % 2] if hp else ())  # one and two dictionary leaves
            out.append(Shape("k_runs_tma", (nl, nk, na, gen, hp), "runs", leaves, RUNS_KEYS_ALL[:nk],
                             aggs + (lp.Count(col(V)),)))
    return out


TILE_K8 = ("labels.a", "labels.b", "labels.c", "labels.d")
TILE_K16 = ("labels.w", "labels.b", "labels.c", "labels.d")
TILE_SUMS = {True: (lp.Sum(col(U)), lp.Sum(col(X))), False: (lp.Sum(col(V)), lp.Sum(col(T)))}
TILE_CUT = col(T).Gt(lit(0))  # about half of every row group


def tile_shapes() -> List[Shape]:
    out = []
    base = (("FROSTGPU_NO_RUNS", "1"),)  # (a plan without keys would take the sorted-run kernel on any part)
    for nk, na, k8, nc in itertools.product(range(5), range(3), B, B):
        inst = (True, True, nk, na, k8, nc)
        if inst in UNREACHABLE["k_tile_agg"]:
            continue
        env = base + ((("FROSTGPU_TA_CARRY", "1"),) if not nc and na == 0 else ())
        leaves = (TILE_CUT,) if (nk + na) % 2 else ()
        out.append(Shape("k_tile_agg", inst, "tiles", leaves, (TILE_K8 if k8 else TILE_K16)[:nk],
                         TILE_SUMS[nc][:na] + (lp.Count(col(V)),), env=env))
    g = base + (("FROSTGPU_TA_GLOBAL", "1"),)
    k2 = TILE_K8[:2]
    generic = [
        ((True, True, -1, -1, False, False), (), k2, (lp.Sum(col(U)), lp.Sum(col(X)), lp.Sum(col(V))), base, "NA = 3"),
        ((True, True, -1, -1, False, False), (TILE_CUT,), TILE_K8, (lp.Sum(col(U)), lp.Sum(col(X)), lp.Sum(col(V)), lp.Sum(col(T))), base, "NA = 4"),
        ((True, False, -1, -1, False, False), (col(F).GtEq(lit(0.0)),), k2, (lp.Sum(col(V)),), base, "float leaf"),
        ((True, False, -1, -1, False, False), (col(V).NotEq(lit(7)),), TILE_K8, (lp.Sum(col(U)),), base, "!= leaf"),
        ((True, False, -1, -1, False, False), (col("labels.b").NotEq(lit("v000001")),), k2, (lp.Sum(col(V)),), base, "dictionary leaf"),
        ((True, False, -1, -1, False, False), (TILE_CUT,), TILE_K8, (lp.Min(col(V)), lp.Max(col(T)), lp.Sum(col(F))), base, "Min / Max / float Sum"),
        ((False, True, -1, -1, False, False), (TILE_CUT,), TILE_K8, (lp.Sum(col(V)), lp.Sum(col(U))), g, "FROSTGPU_TA_GLOBAL"),
        ((False, True, -1, -1, False, False), (), ("labels.e", "labels.c"), (lp.Sum(col(V)),), base, "32-bit codes: table over 227 KB"),
        ((False, False, -1, -1, False, False), (TILE_CUT,), k2, (lp.Min(col(V)), lp.Max(col(U))), g, "FROSTGPU_TA_GLOBAL"),
        ((False, False, -1, -1, False, False), (col(F).Lt(lit(0.0)),), ("labels.e",), (lp.Max(col(T)), lp.Sum(col(F))), base, "32-bit codes: table over 227 KB"),
    ]
    for inst, leaves, keys, aggs, env, note in generic:
        out.append(Shape("k_tile_agg", inst, "tiles", leaves, keys, aggs + (lp.Count(col(V)),), env=env, note=note))
    return out


# take table: `value` is a permutation of 0 .. n (n = TAKE_ROWS) without TAKE_ABSENT, shuffled over the whole part, so
# every row group holds 0 and n and no range leaf on `value` is decided or pruned by the statistics (a dictionary leaf
# keeps the take path only when no row group is pruned); `timestamp` is 0 .. n - 1 in order
TAKE_ROWS, TAKE_RG, TAKE_ABSENT = 3 * 8192, 8192, 777
TAKE_OUT_COLS = (T, V, W, F)
TAKE_SELECT = {"none": col(V).Eq(lit(TAKE_ABSENT)), "one": col(V).Eq(lit(12_345)),
               "half": col(V).Lt(lit(TAKE_ROWS // 2)), "all": col(V).LtEq(lit(TAKE_ROWS))}
TAKE_TS = col(T).GtEq(lit(TAKE_RG // 2))  # row group 0 filtered row by row, the others decided by statistics
TAKE_DICT = (col("labels.a").NotEq(lit("v000001")), col("labels.b").Eq(lit("v000000")))


def take_shapes() -> List[Shape]:
    """Every (NL, NO, HP): 0-2 range leaves x 0-2 dictionary leaves x 1-4 projected columns; the range leaf on
    `value` rotates over selecting nothing, one row, about half and everything."""
    out = []
    sels = ("none", "one", "half", "all")
    for i, (nl, no, n_dict) in enumerate(itertools.product(range(3), range(1, 5), range(3))):
        sel = sels[i % 4] if nl else "-"
        leaves = ((TAKE_SELECT[sel],) if nl >= 1 else ()) + ((TAKE_TS,) if nl == 2 else ()) + TAKE_DICT[:n_dict]
        out.append(Shape("k_take_write", (nl, no, n_dict > 0), "take", leaves, out=TAKE_OUT_COLS[:no], note=sel))
    return out


PREFIX_CARD = {"labels.a": 3, "labels.b": 4, "labels.c": 2}
PREFIX_RUNS = {"labels.a": 8, "labels.b": 32, "labels.c": PREFIX_MANY_RUNS}  # runs per row group


def prefix_shapes() -> List[Shape]:
    facts = {"runs": PREFIX_RUNS, "rows": PREFIX_RG, "row_groups": PREFIX_RGS, "card": PREFIX_CARD}
    sums = (lp.Sum(col(V)), lp.Sum(col(T)), lp.Count(col(V)))
    out = []
    for keys in (("labels.c",), ("labels.a", "labels.b"), ("labels.a",), ()):
        s = Shape("k_runs_prefix", (), "prefix", (), keys, sums, facts=facts)
        out.append(Shape("k_runs_prefix", expected_instance("k_runs_prefix", s), "prefix", (), keys, sums, facts=facts))
    return out


# fast table: parts 0..3 hold keys labels.a..c, a..b, a, none (NK = 3 - part); row group r of every part leaves
# 2 - r of the two leaves undecided (the first leaf stays undecided longest)
FAST_KEYS_ALL = ("labels.a", "labels.b", "labels.c")
FAST_PARTS, FAST_RGS_PER_PART, FAST_RG = 4, 3, 4096
FAST_PLANS = {  # (NA, tight) -> (leaves, stored aggregates)
    (0, True): ((col(V).GtEq(lit(0)), col(T).GtEq(lit(0))), ()),
    (1, True): ((col(V).GtEq(lit(0)), col(T).GtEq(lit(0))), (lp.Sum(col(V)),)),
    (2, True): ((col(V).GtEq(lit(0)), col(T).GtEq(lit(0))), (lp.Sum(col(V)), lp.Sum(col(T)))),
    (0, False): ((col(F).GtEq(lit(0.0)), col(T).GtEq(lit(0))), ()),
    (1, False): ((col(V).GtEq(lit(0)), col(T).GtEq(lit(0))), (lp.Min(col(V)),)),
    (2, False): ((col(V).GtEq(lit(0)), col(T).GtEq(lit(0))), (lp.Max(col(T)), lp.Sum(col(F)))),
}
FAST_SWITCHES = (("FROSTGPU_NO_RUNS", "1"), ("FROSTGPU_NO_TILE", "1"))


def fast_shapes() -> List[Shape]:
    """One plan per (NA, tight) covers every (NL, NK) of the table's row groups: the shapes list each tuple with the
    row group (part, row group) that selects it."""
    out = []
    for (na, tight), (leaves, stored) in FAST_PLANS.items():
        for part, r in itertools.product(range(FAST_PARTS), range(FAST_RGS_PER_PART)):
            facts = {"decided": (r >= 2, r >= 1), "keys_present": FAST_KEYS - part, "row_group": (part, r)}
            s = Shape("fast_pass", (), "fast", leaves, FAST_KEYS_ALL, stored + (lp.Count(col(V)),), env=FAST_SWITCHES, facts=facts)
            out.append(Shape("fast_pass", expected_instance("fast_pass", s), "fast", leaves, FAST_KEYS_ALL, s.aggs,
                             env=FAST_SWITCHES, facts=facts))
    return out


def shapes(kernel: str) -> List[Shape]:
    if kernel == "k_runs_tma":
        return runs_shapes()
    if kernel == "k_tile_agg":
        return tile_shapes()
    if kernel == "k_take_write":
        return take_shapes()
    if kernel == "k_take_count":  # every take plan launches both kernels: count (NL, HP), write (NL, NO, HP)
        return [Shape("k_take_count", (s.instance[0], s.instance[2]), s.table, s.leaves, out=s.out, note=s.note) for s in take_shapes()]
    if kernel == "k_runs_prefix":
        return prefix_shapes()
    if kernel == "fast_pass":
        return fast_shapes()
    raise KeyError(kernel)
