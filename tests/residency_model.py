"""A plain model of lazily built column images (no engine or oracle code): seeded fixture parts that share one schema,
an exact reference answer over any set of visible parts, a bank of plans aimed at known scan kernels, and a seeded
generator of operation sequences (puts, queries, decodes, drops, corrupted parts, kernel switches).

Schema: string columns stored as dictionary (`s_dict`), PLAIN (`s_plain`), DELTA_LENGTH_BYTE_ARRAY (`s_dlba`),
DELTA_BYTE_ARRAY (`s_dba`) and dictionary with a PLAIN fallback (`s_fallback`); `timestamp` (sorted, PLAIN or
DELTA_BINARY_PACKED); `value` (int64, PLAIN or DELTA_BINARY_PACKED, full-range in some parts so that Sum wraps);
`floatvalue` (nullable, multiples of 1/8, so that every order of addition gives the same sum); the dynamic label
`labels.x`, which only some parts have.

The reference reads each part's bytes with pyarrow and aggregates with tests/numeric_edges.py (numpy and Python ints):
Sum(int64) wraps modulo 2^64, Count counts rows, Min / Max exactly, NULL keys form their own group, a column a part
lacks is NULL there, and filter-only plans keep row order (parts in the order they were put)."""
import dataclasses
import functools
import io
import random
from typing import Dict, List, Optional, Tuple

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq

from frostdb_b200 import logicalplan as lp
from tests import numeric_edges as ne

STRINGS = ["s_dict", "s_plain", "s_dlba", "s_dba", "s_fallback"]
LABEL = "labels.x"
DICT_COLS = ["s_dict", "s_fallback", LABEL]
STRING_ENCODING = {"s_plain": "PLAIN", "s_dlba": "DELTA_LENGTH_BYTE_ARRAY", "s_dba": "DELTA_BYTE_ARRAY"}
DBP = "DELTA_BINARY_PACKED"
FALLBACK_LIMIT = 4096  # dictionary page limit of the writer: s_fallback's dictionary outgrows it, s_dict's never does
LENGTHS = [0, 1, 7, 8, 31, 32, 33, 64]  # XXH64 tails and 32-byte stripes
EDGE_RGS = [1, 31, 32, 33, 255, 256, 257, 4097]
EDGE_DISTINCT = [1, 2, 3, 33, 255, 256, 257, 4097]  # s_plain: code widths 0, 1, 2, 6, 8, 8, 9, 13
WIDE_RGS = [300, 66000, 4096]
WIDE_DISTINCT = 65537  # s_plain of the wide part's second row group: 17-bit codes
I64_MIN, I64_MAX = ne.I64_MIN, ne.I64_MAX


@dataclasses.dataclass(frozen=True)
class Spec:
    """A fixture part.  key: how s_dict is laid out ("runs" of `run` rows, "random", or the edge layouts); rgs: the
    row group sizes."""
    name: str
    seed: int
    key: str
    rgs: Tuple[int, ...]
    ts_dbp: bool = False
    value_dbp: bool = False
    wrap: bool = False
    label: bool = False
    run: int = 128


SPECS = [
    Spec("sorted_a", 1, "runs", (2048, 2048), ts_dbp=True, label=True),
    Spec("sorted_b", 2, "runs", (2048, 2048), wrap=True),
    Spec("unsorted_a", 3, "random", (2048, 2048), value_dbp=True, label=True),
    Spec("short_runs", 4, "runs", (1024, 1024, 1024), ts_dbp=True, value_dbp=True, wrap=True, run=3),
    Spec("sorted_c", 5, "runs", (1024, 1024, 1024, 1024), ts_dbp=True, label=True, run=256),
    Spec("edge", 6, "edge", tuple(EDGE_RGS), value_dbp=True, label=True),
    Spec("wide", 7, "wide", tuple(WIDE_RGS)),
]
SPEC_BY_NAME = {s.name: s for s in SPECS}
WALK_PARTS = [s.name for s in SPECS if s.name != "wide"]  # (the wide part is 70 000 rows: its own tests only)


# ---- fixture parts -----------------------------------------------------------------------------------------------
def _shared(col: str, n: int) -> List[str]:
    """Values every part draws on: long shared prefixes (front coding)."""
    return [f"/srv/app/{col}/module_{i % 7:02d}/frame_{i}" for i in range(n)]


def _own(spec: Spec, col: str, n: int) -> List[str]:
    """Values only this part has: every put can grow the dictionaries."""
    return [f"{spec.name}/{col}/{i}" for i in range(n)]


def _edge_value(k: int) -> str:
    """The k-th distinct edge value: hex digits then dots, at the lengths of LENGTHS where the digits fit."""
    s = f"{k:x}" if k else ""
    return s + "." * max(0, LENGTHS[k % len(LENGTHS)] - len(s))


def _edge_dba(rng, n: int) -> List[str]:
    """Values equal to the one before, or a prefix of the one after, or new."""
    out, prev = [], ""
    for _ in range(n):
        r = rng.random()
        if r < 0.3:
            v = prev
        elif r < 0.6 and len(prev) < 80:
            v = prev + "abcdefgh"[int(rng.integers(0, 8))]
        else:
            v = _edge_value(int(rng.integers(0, 300)))
        out.append(v)
        prev = v
    return out


@functools.lru_cache(maxsize=None)
def table_of(name: str) -> pa.Table:
    spec = SPEC_BY_NAME[name]
    rng = np.random.default_rng(1000 + spec.seed)
    n = sum(spec.rgs)
    pick = lambda pool, m: [pool[int(i)] for i in rng.integers(0, len(pool), m)]
    nulls = lambda p: rng.random(n) < p
    cols: Dict[str, object] = {}
    if spec.key == "runs":
        pool = sorted(_shared("s_dict", 40) + _own(spec, "s_dict", 10))
        runs = [pool[int(i)] for i in np.sort(rng.integers(0, len(pool), (n + spec.run - 1) // spec.run))]
        cols["s_dict"] = [runs[i // spec.run] for i in range(n)]
    elif spec.key == "wide":
        r0, r1, r2 = WIDE_RGS
        w = [f"w/{i}" for i in range(r1)]
        cols["s_dict"] = pick(w[:200], r0) + w + pick(w[256:60000], r2)
    else:
        cols["s_dict"] = pick(_shared("s_dict", 40) + _own(spec, "s_dict", 10), n)
    if spec.key == "edge":
        plain, dlba, dba = [], [], []
        for rows, d in zip(EDGE_RGS, EDGE_DISTINCT):
            vals = [_edge_value(k) for k in range(d)]
            plain += vals + pick(vals, rows - d)  # every one of the d values occurs
            dlba += pick(vals[::-1], rows)
            dba += _edge_dba(rng, rows)
        cols["s_plain"], cols["s_dlba"], cols["s_dba"] = plain, dlba, dba
    elif spec.key == "wide":
        r0, r1, r2 = WIDE_RGS
        vals = [f"{k:x}" for k in range(WIDE_DISTINCT)]
        cols["s_plain"] = pick(vals[:50], r0) + vals + pick(vals, r1 - WIDE_DISTINCT) + pick(vals[:5000], r2)
        cols["s_dlba"] = pick(_shared("s_dlba", 300), n)
        cols["s_dba"] = sorted(pick(_shared("s_dba", 500), n))
    else:
        cols["s_plain"] = pick(_shared("s_plain", 150) + _own(spec, "s_plain", 30), n)
        cols["s_dlba"] = pick(_shared("s_dlba", 300) + _own(spec, "s_dlba", 40), n)
        cols["s_dba"] = sorted(pick(_shared("s_dba", 500) + _own(spec, "s_dba", 60), n))
    cols["s_fallback"] = pick(_shared("s_fallback", 1500) + _own(spec, "s_fallback", 200), n)
    for c, p in (("s_plain", 0.0 if spec.key in ("edge", "wide") else 0.05), ("s_dba", 0.08)):  # (edge widths stay exact)
        cols[c] = [None if x else v for v, x in zip(cols[c], nulls(p))]
    if spec.label:
        cols[LABEL] = [None if x else v for v, x in zip(pick(["a", "b", "c"], n), nulls(0.2))]
    base = (spec.seed + 1) * 10_000_000
    cols["timestamp"] = pa.array(base + 3 * np.arange(n, dtype=np.int64))
    if spec.wrap:
        cols["value"] = pa.array(rng.integers(I64_MAX // 4, I64_MAX, n, dtype=np.int64, endpoint=True) * rng.choice([-1, 1], n))
    else:
        cols["value"] = pa.array(rng.integers(-1000, 1000, n, dtype=np.int64))
    cols["floatvalue"] = pa.array(rng.integers(-4000, 4000, n) / 8.0, mask=nulls(0.1))
    arrays = {k: (v if isinstance(v, pa.Array) else pa.array(v, type=pa.string())) for k, v in cols.items()}
    fields = [pa.field(k, arrays[k].type, nullable=k in ("s_plain", "s_dba", LABEL, "floatvalue")) for k in sorted(arrays)]
    meta = {"dynamic_columns": "labels:x" if spec.label else ""}
    return pa.Table.from_arrays([arrays[f.name] for f in fields], schema=pa.schema(fields)).replace_schema_metadata(meta)


def row_group_bounds(name: str) -> List[Tuple[int, int]]:
    out, b = [], 0
    for n in SPEC_BY_NAME[name].rgs:
        out.append((b, b + n))
        b += n
    return out


def encodings(buf: bytes) -> Dict[str, List[set]]:
    """Per column, the encodings the footer lists for each row group."""
    md = pq.ParquetFile(io.BytesIO(buf)).metadata
    names = [md.schema.column(i).path for i in range(md.num_columns)]
    return {c: [set(md.row_group(g).column(i).encodings) for g in range(md.num_row_groups)] for i, c in enumerate(names)}


@functools.lru_cache(maxsize=None)
def file_of(name: str) -> bytes:
    """The part's Parquet bytes: one row group per entry of its spec's `rgs`.  Asserts the layouts it claims."""
    spec = SPEC_BY_NAME[name]
    t = table_of(name)
    enc = dict(STRING_ENCODING, floatvalue="PLAIN", timestamp=DBP if spec.ts_dbp else "PLAIN", value=DBP if spec.value_dbp else "PLAIN")
    dict_cols = [c for c in DICT_COLS if c in t.column_names]
    sink = io.BytesIO()
    limit = 1 << 28 if spec.key == "wide" else FALLBACK_LIMIT
    with pq.ParquetWriter(sink, t.schema, compression="NONE", use_dictionary=dict_cols, column_encoding=enc,
                          dictionary_pagesize_limit=limit, data_page_size=1 << 16, store_schema=False) as w:
        for lo, hi in row_group_bounds(name):
            w.write_table(t.slice(lo, hi - lo), row_group_size=hi - lo)
    buf = sink.getvalue()
    e = encodings(buf)
    assert len(e["timestamp"]) == len(spec.rgs)
    for c, want in enc.items():
        for g in e[c]:
            assert want in g, (name, c, want, g)
            assert not g & {"RLE_DICTIONARY", "PLAIN_DICTIONARY"}, (name, c, g)
    for c in dict_cols:
        assert all("RLE_DICTIONARY" in g for g in e[c]), (name, c)
    if spec.key != "wide":  # the fallback: distinct values far beyond what a dictionary page of the limit holds
        for lo, hi in row_group_bounds(name):
            distinct = set(t.column("s_fallback").slice(lo, hi - lo).to_pylist())
            assert hi - lo < 1000 or sum(len(v) + 4 for v in distinct) > 4 * FALLBACK_LIMIT, name
    return buf


def record_of(name: str) -> pa.RecordBatch:
    """The part as an Arrow record (strings as binary, as the Go side hands labels over)."""
    t = table_of(name).combine_chunks()
    cols = [t.column(n).chunk(0) for n in t.column_names]
    cols = [c.cast(pa.binary()) if pa.types.is_string(c.type) else c for c in cols]
    return pa.RecordBatch.from_arrays(cols, names=t.column_names)


def key_widths(name: str, column: str) -> List[int]:
    """Per row group, the bit width of chunk-local codes over the chunk's distinct non-null values."""
    t = table_of(name)
    out = []
    for lo, hi in row_group_bounds(name):
        d = len({v for v in t.column(column).slice(lo, hi - lo).to_pylist() if v is not None})
        out.append(max(d - 1, 0).bit_length())
    return out


# ---- the reference -----------------------------------------------------------------------------------------------
ALL_COLUMNS = sorted(STRINGS + [LABEL, "timestamp", "value", "floatvalue"])


@functools.lru_cache(maxsize=None)
def physical(name: str) -> Dict[str, np.ndarray]:
    """The part as the reference reads it, from pyarrow's read of its bytes: strings as object arrays (None = NULL,
    also for a column the part lacks), nullable floats as raw slots (NULL = 0.0, ne.physical)."""
    t = pq.read_table(io.BytesIO(file_of(name)))
    n = t.num_rows
    out = {}
    for c in ALL_COLUMNS:
        if c not in t.column_names:
            out[c] = np.array([None] * n, dtype=object)
            continue
        a = t.column(c).combine_chunks()
        if pa.types.is_dictionary(a.type):
            a = a.dictionary_decode()
        if pa.types.is_string(a.type):
            out[c] = np.array(a.to_pylist(), dtype=object)
        else:
            out.update(ne.physical({c: a}))
    return out


def reference(plan: "Plan", parts: List[str]):
    """The plan's answer over `parts` (in the order they were put): {key: aggregates}, a set of Distinct tuples or the
    filter-only rows."""
    phys = [physical(p) for p in parts]
    if plan.kind == "agg":
        return ne.reference(phys, plan.filt, plan.keys, plan.aggs)
    if plan.kind == "distinct":
        out = set()
        for cols in phys:
            sel = ne.selection(cols, plan.filt)
            out |= {r for r in zip(*[cols[k][sel].tolist() for k in plan.keys]) if r != (None,) * len(plan.keys)}
        return out
    rows = []
    for cols in phys:
        sel = np.flatnonzero(ne.selection(cols, plan.filt))
        got = []
        for c in plan.keys:
            v = cols[c][sel].tolist()
            if c + "#valid" in cols:
                v = [x if ok else None for x, ok in zip(v, cols[c + "#valid"][sel].tolist())]
            got.append(v)
        rows.extend(zip(*got))
    return rows


def float_groups(plan: "Plan", parts: List[str]) -> set:
    """Keys of the aggregate plan's groups that select at least one non-NULL floatvalue."""
    out = set()
    for cols in (physical(p) for p in parts):
        sel = ne.selection(cols, plan.filt) & cols["floatvalue#valid"] if "floatvalue#valid" in cols else ne.selection(cols, plan.filt)
        keys = [ne._key_values(k, {c: np.asarray(v)[sel] for c, v in cols.items()}) for k in plan.keys]
        out |= set(zip(*keys)) if plan.keys else ({()} if sel.any() else set())
    return out


# ---- the plan bank -----------------------------------------------------------------------------------------------
V, T, F = lp.Col("value"), lp.Col("timestamp"), lp.Col("floatvalue")
TS_SPLIT = 4 * 10_000_000  # timestamps of parts with seed >= 3 (unsorted_a and later) lie above it


@dataclasses.dataclass(frozen=True)
class Plan:
    """kind: "agg", "distinct" or "rows" (filter-only; `keys` are the projected columns).  kernel: the kernel the
    default switches send the sorted parts' row groups to (the others go to k_tile_agg or k_scan).  cached: a dense
    aggregate whose repeated Execute reuses the compiled plan's device state and copies nothing."""
    name: str
    kind: str
    keys: Tuple[str, ...]
    aggs: Tuple = ()
    filt: Optional[lp.Expr] = None
    kernel: str = ""
    cached: bool = False


def bank() -> List[Plan]:
    s = lambda c: lp.Col(c)
    lit_dict = _shared("s_dict", 40)[3]
    return [
        Plan("prefix", "agg", ("s_dict",), (lp.Sum(V), lp.Count(V)), None, "k_runs_prefix", True),
        Plan("runs", "agg", ("s_dict",), (lp.Sum(V), lp.Min(V), lp.Max(V)), T.Gt(lp.Literal(2 * 10_000_000 + 5000)), "k_runs_tma", True),
        Plan("tile", "agg", ("s_plain", LABEL), (lp.Sum(V), lp.Count(V), lp.Max(V)), V.Gt(lp.Literal(-500)), "k_tile_agg", True),
        Plan("scan_fast", "agg", ("s_dba",), (lp.Sum(F), lp.Count(V)), V.Lt(lp.Literal(800)), "k_scan", True),
        Plan("scan_hash", "agg", ("value",), (lp.Count(V), lp.Sum(F)),
             lp.Or(s("s_fallback").Eq(lp.Literal(_shared("s_fallback", 1500)[7])), V.Lt(lp.Literal(-900))), "k_scan"),
        Plan("hash_strings", "agg", ("s_plain", "s_dlba", "s_fallback"), (lp.Count(V), lp.Min(T)), None, "k_scan"),
        Plan("pruned", "agg", ("s_dlba",), (lp.Sum(V), lp.Count(V), lp.Min(T)),
             lp.And(T.Lt(lp.Literal(TS_SPLIT)), s("s_dlba").Eq(lp.Literal(_shared("s_dlba", 300)[11]))), "k_tile_agg", True),
        Plan("take", "rows", ("timestamp", "value", "floatvalue"), (), lp.And(T.GtEq(lp.Literal(TS_SPLIT)), V.Gt(lp.Literal(900))), "k_take"),
        Plan("tile_dict_leaf", "agg", ("s_dlba",), (lp.Sum(V), lp.Count(V)), s("s_dict").NotEq(lp.Literal(lit_dict)), "k_tile_agg", True),
        Plan("take_dict", "rows", ("timestamp", "value"), (), s("s_dict").NotEq(lp.Literal(lit_dict)), "k_take"),
        Plan("rows", "rows", ("timestamp", "s_plain", "s_dba", LABEL), (), s("s_dict").Eq(lp.Literal(lit_dict)), "k_rows"),
        Plan("distinct", "distinct", ("s_fallback",), (), None, "distinct"),
        Plan("distinct_pair", "distinct", ("s_dict", "s_dlba"), (), s("s_dba").NotEq(lp.Literal(_shared("s_dba", 500)[0])), "distinct"),
    ]


# ---- operation sequences -----------------------------------------------------------------------------------------
HOWS = ("eager", "borrow", "arrow")
SWITCHES = ("FROSTGPU_NO_PREFIX", "FROSTGPU_NO_RUNS")
CORRUPT_CASES = ("bit_width", "miniblock_overrun", "count")  # tests/delta_int64.py: refused on the host at residency


def sequence(seed: int, steps: int, parts=tuple(WALK_PARTS), max_visible: int = 4) -> List[tuple]:
    """A deterministic walk of `steps` operations:
    ("put", part, how), ("query", plan index, "fresh" | "prepared"), ("decode", part, column), ("drop", part),
    ("corrupt", case), ("switch", name, on).  A part is visible at most once; drops and decodes name a visible part; a
    prepared query re-runs a plan run before."""
    rng = random.Random(seed)
    n_plans = len(bank())
    visible: List[str] = []
    ran: List[int] = []
    switches = {k: False for k in SWITCHES}
    out = []
    while len(out) < steps:
        r = rng.random()
        if not visible or (r < 0.25 and len(visible) < max_visible):
            p = rng.choice([x for x in parts if x not in visible])
            visible.append(p)
            out.append(("put", p, rng.choice(HOWS)))
        elif r < 0.65:
            if ran and rng.random() < 0.4:
                out.append(("query", rng.choice(ran), "prepared"))
            else:
                i = rng.randrange(n_plans)
                ran.append(i)
                out.append(("query", i, "fresh"))
        elif r < 0.75:
            p = rng.choice(visible)
            out.append(("decode", p, rng.choice(table_of(p).column_names)))
        elif r < 0.85 and len(visible) > 1:
            p = rng.choice(visible)
            visible.remove(p)
            out.append(("drop", p))
        elif r < 0.92:
            out.append(("corrupt", rng.choice(CORRUPT_CASES)))
        else:
            k = rng.choice(SWITCHES)
            switches[k] = not switches[k]
            out.append(("switch", k, switches[k]))
    return out
