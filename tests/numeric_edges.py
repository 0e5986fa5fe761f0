"""Numeric edge cases for every scan path: datasets whose values sit at the ends of int64, around 2^53 and on the IEEE
specials, and a plain reference of the physical plan's semantics written with numpy and Python ints.  The reference
shares nothing with the engine or the oracle; its rules are the few lines of `_leaf_mask`, `_aggregate` and
`same_value`:

- a leaf never selects NULL; `x != NaN` holds for every non-NULL x (arrow compute);
- an int64 column against a float literal compares float(x) (round to nearest even), as the oracle and arrow do;
- Sum(int64) wraps modulo 2^64; Sum(float64) adds in row order; Count counts rows;
- Min / Max follow Go's sequential rule (`if v < m`, the first value seeds m);
- filter-only plans return the selected rows in insertion order.

The datasets keep every float Sum independent of the summation order (dyadic values k / 1024 whose partial sums stay
below 2^53 ulps, specials whose result is the same in every order) and never put NaN first in a group within a row
group, so the sequential Min / Max equals "NaN is never selected" for any merge order.  Keys are non-null dictionary
labels."""
from __future__ import annotations

import math
import struct
from typing import Dict, List, Sequence

import numpy as np

from frostdb_b200 import dynparquet as dp
from frostdb_b200 import logicalplan as lp
from tests.util import label_values

I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
DBL_MAX = np.finfo(np.float64).max
DENORM_MIN = 5e-324
NAN, INF = float("nan"), float("inf")
RG = 4096
KA, KB = 4, 6  # labels.a x labels.b: 24 groups

# (lo, hi) of `value` per row group, both ends present: frame-of-reference widths 8, 16, 32, 64, 8 (where double(x)
# rounds) and 8 bits, at and around the ends of int64
INT_CHUNKS = [(-7, 248), (I64_MIN, I64_MIN + 65_535), (I64_MAX - (1 << 32) + 1, I64_MAX), (I64_MIN, I64_MAX),
              ((1 << 53) - 64, (1 << 53) + 64), (-1, 0)]
EDGE_LITERALS = [I64_MIN, I64_MIN + 1, -1, 0, I64_MAX - 1, I64_MAX]
OPS = [lp.OpEq, lp.OpNotEq, lp.OpLt, lp.OpLtEq, lp.OpGt, lp.OpGtEq]


def leaf(col: str, op: int, value) -> lp.Expr:
    return lp.BinaryExpr(lp.Col(col), op, lp.Literal(value))


def chunk_literals(chunks=INT_CHUNKS) -> List[int]:
    """min - 1, min, max, max + 1 of every chunk (inside int64)."""
    out = set()
    for lo, hi in chunks:
        out.update(v for v in (lo - 1, lo, hi, hi + 1) if I64_MIN <= v <= I64_MAX)
    return sorted(out)


# ---- datasets ----------------------------------------------------------------------------------------------------
def _chunk_values(rng, lo: int, hi: int, n: int) -> np.ndarray:
    v = [lo + int(x) % (hi - lo + 1) for x in rng.integers(0, 1 << 62, n, dtype=np.int64)]
    v[int(rng.integers(0, n))] = lo
    v[int(rng.integers(0, n))] = hi
    return np.array(v, dtype=np.int64)


def float_column(g: np.ndarray, seed: int, rg: int = RG, part: int = 0) -> np.ndarray:
    """floatvalue by flavour of the group (g % 6), in physical row order:
    0 dyadic values (|k| < 2^40) and +-0.0; 1 dyadic values and NaN; 2 non-negative dyadic values and two DBL_MAX
    (Sum +inf); 3 dyadic values, +inf and -DBL_MAX (Sum +inf); 4 dyadic values, +inf, -inf and NaN (Sum NaN);
    5 +-0.0 and 5e-324 (exact subnormal Sum).  In groups with NaN the first two rows of every row group are 0.5 and
    -0.25, so no single `!=` leaf leaves a NaN first.  The specials of a group go into one part of a table only
    (`part` 0 takes the groups with (g // 6) even, `part` 1 the others): two parts that both held +inf and -DBL_MAX
    would put two -DBL_MAX in one group, and -DBL_MAX + -DBL_MAX = -inf makes the Sum depend on the order."""
    rng = np.random.default_rng(seed)
    n = len(g)
    k = rng.integers(-(1 << 20), 1 << 20, n)
    big = rng.random(n) < 0.01
    k[big] = rng.integers(-(1 << 40) + 1, 1 << 40, int(big.sum()))
    f = k.astype(np.float64) / 1024.0
    fl = g % 6
    f[(fl == 0) & (rng.random(n) < 0.05)] = 0.0
    f[(fl == 0) & (rng.random(n) < 0.05)] = -0.0
    f[fl == 2] = np.abs(f[fl == 2])
    z = fl == 5
    f[z] = np.where(rng.random(int(z.sum())) < 0.5, np.where(rng.random(int(z.sum())) < 0.5, -0.0, 0.0), DENORM_MIN)
    for grp in np.unique(g):
        specials = {1: [NAN] * 5, 2: [DBL_MAX, DBL_MAX], 3: [INF, -DBL_MAX], 4: [INF, -INF, NAN, NAN]}.get(int(grp % 6), [])
        if not specials or (grp // 6) % 2 != part:
            continue
        lead = set()  # the first two rows of the group in every row group
        for r0 in range(0, n, rg):
            lead.update((r0 + np.flatnonzero(g[r0:r0 + rg] == grp))[:2].tolist())
        if grp % 6 in (1, 4):
            for r in lead:
                f[r] = 0.5 if r == min(x for x in lead if x // rg == r // rg) else -0.25
        rest = np.array(sorted(set(np.flatnonzero(g == grp).tolist()) - lead), dtype=np.int64)
        assert len(rest) >= 2 * len(specials)
        f[rng.choice(rest, len(specials), replace=False)] = specials
    return f


def int_part(chunks, seed: int, *, sort: bool, t0: int = 0, rg: int = RG, part: int = 0) -> Dict[str, object]:
    """One part whose row group k holds `rg` rows with `value` in chunks[k] (both ends present).  Sorted parts are
    generated in the order compaction writes them (keys sorted, timestamps rising), so row group k is rows
    [k * rg, (k + 1) * rg) of the columns as given; unsorted parts are written as they are (sort=False).  `part`: the
    part's index in its table (see float_column)."""
    n = rg * len(chunks)
    rng = np.random.default_rng(seed)
    g = rng.integers(0, KA * KB, n)
    if sort:
        g = np.sort(g)
    value = np.concatenate([_chunk_values(rng, lo, hi, rg) for lo, hi in chunks])
    return {
        "example_type": (np.zeros(n, np.int32), ["cpu"]),
        "stacktrace": (rng.integers(0, 5, n).astype(np.int32), [f"stack{i:02d}" for i in range(5)]),
        "timestamp": t0 + np.arange(n, dtype=np.int64),
        "value": value,
        "labels.a": ((g // KB).astype(np.int32), label_values(KA)),
        "labels.b": ((g % KB).astype(np.int32), label_values(KB)),
        "floatvalue": float_column(g, seed + 1, rg, part),
    }


def write(cols: Dict[str, object], *, sort: bool, stats: bool = True, rg: int = RG) -> bytes:
    """The part as Parquet.  A sorted part must already be in compaction order (asserted), so the physical order is
    the order of `cols` either way."""
    schema = dp.SampleDefinitionWithFloat() if "floatvalue" in cols else dp.SampleDefinition()
    if sort:
        n = len(cols["timestamp"])
        assert np.array_equal(dp.sort_permutation(schema, cols, n), np.arange(n))
    return dp.write_part(schema, cols, sort=False, row_group_size=rg, write_statistics=stats)


def wrap_part(n: int, seed: int, *, t0: int = 0, ka: int = KA, kb: int = KB, used=None) -> Dict[str, object]:
    """Unsorted part with `value` spread over all of int64: group sums cross +-2^63 many times.  ka x kb labels in
    the dictionaries; `used` = (na, nb) restricts the rows to the first na x nb of them (hash-table mode with few
    groups)."""
    rng = np.random.default_rng(seed)
    na, nb = used or (ka, kb)
    a = rng.integers(0, na, n).astype(np.int32)
    b = rng.integers(0, nb, n).astype(np.int32)
    value = rng.integers(I64_MIN, I64_MAX, n, dtype=np.int64, endpoint=True)
    value[:: 97] = I64_MAX
    value[1:: 89] = I64_MIN
    return {
        "example_type": (np.zeros(n, np.int32), ["cpu"]),
        "stacktrace": (rng.integers(0, 3, n).astype(np.int32), [f"stack{i:02d}" for i in range(3)]),
        "timestamp": t0 + np.arange(n, dtype=np.int64),
        "value": value,
        "labels.a": (a, label_values(ka)),
        "labels.b": (b, label_values(kb)),
    }


DIVISORS = [0, 1, -1, 2, -2, 3, -3, I64_MIN, I64_MAX]


def expr_part(seed: int, *, sort: bool, t0: int = 0, part: int = 0) -> Dict[str, object]:
    """A part for arithmetic aggregate inputs and computed keys: int_part's `value` over INT_CHUNKS and its labels,
    and `floatvalue` with ~3 % NULL rows (none on a special, so float_column's order rules still hold).  Sorted parts
    keep timestamps t0, t0 + 1, ... (negative for t0 < 0: time buckets on both sides of 0); unsorted parts draw
    `timestamp` from DIVISORS (two thirds of the rows) and from all of int64, as the second operand of `value`."""
    import pyarrow as pa
    cols = int_part(INT_CHUNKS, seed, sort=sort, t0=t0, part=part)
    rng = np.random.default_rng(seed + 7)
    n = len(cols["timestamp"])
    if not sort:
        ts = rng.integers(I64_MIN, I64_MAX, n, dtype=np.int64, endpoint=True)
        pick = rng.random(n) < 2 / 3
        ts[pick] = np.array(DIVISORS, dtype=np.int64)[rng.integers(0, len(DIVISORS), int(pick.sum()))]
        ts[np.flatnonzero(cols["value"] == I64_MIN)[::2]] = -1  # INT64_MIN / -1
        cols["timestamp"] = ts
    f = cols["floatvalue"]
    nulls = (rng.random(n) < 0.03) & np.isfinite(f) & (np.abs(f) < 2.0 ** 41) & (f != DENORM_MIN)
    cols["floatvalue"] = pa.array(f, mask=nulls)
    return cols


def encoded_parts(seed: int) -> List[tuple]:
    """`value` in the encodings NumReader reads besides a required PLAIN chunk: an optional PLAIN chunk with NULLs,
    and an RLE_DICTIONARY chunk (CK_DICT64) with NULLs.  [(name, columns, Parquet bytes)], written by pyarrow with
    labels.a / labels.b dictionary-encoded; `value` keeps INT_CHUNKS' ends and a real 0 next to its NULLs (a NULL
    int64 key groups with 0)."""
    import io

    import pyarrow as pa
    import pyarrow.parquet as pq
    out = []
    for i, (name, dict_value) in enumerate((("nullable_plain", False), ("dict64", True))):
        rng = np.random.default_rng(seed + i)
        n = RG * 3
        g = rng.integers(0, KA * KB, n)
        # the dictionary page holds at most a few thousand distinct values: draw from a pool that has both ends
        pool = np.concatenate([_chunk_values(rng, lo, hi, 300) for lo, hi in INT_CHUNKS] + [np.zeros(1, np.int64)])
        v = pool[rng.integers(0, len(pool), n)]
        v[:: 101] = 0
        nulls = rng.random(n) < 0.05
        ts = rng.integers(I64_MIN, I64_MAX, n, dtype=np.int64, endpoint=True)
        pick = rng.random(n) < 2 / 3
        ts[pick] = np.array(DIVISORS, dtype=np.int64)[rng.integers(0, len(DIVISORS), int(pick.sum()))]
        cols = {
            "labels.a": ((g // KB).astype(np.int32), label_values(KA)),
            "labels.b": ((g % KB).astype(np.int32), label_values(KB)),
            "timestamp": ts,
            "value": pa.array(v, mask=nulls),
        }
        arrays = [pa.DictionaryArray.from_arrays(pa.array(cols[c][0]), pa.array(cols[c][1])) for c in ("labels.a", "labels.b")]
        t = pa.Table.from_arrays(arrays + [pa.array(ts), cols["value"]], schema=pa.schema([
            pa.field("labels.a", arrays[0].type, nullable=True), pa.field("labels.b", arrays[1].type, nullable=True),
            pa.field("timestamp", pa.int64(), nullable=False), pa.field("value", pa.int64(), nullable=True)]))
        t = t.replace_schema_metadata({"dynamic_columns": "labels:a,b"})
        sink = io.BytesIO()
        pq.write_table(t, sink, compression="NONE", use_dictionary=["labels.a", "labels.b"] + (["value"] if dict_value else []),
                       column_encoding=None if dict_value else {"timestamp": "PLAIN", "value": "PLAIN"},
                       data_page_version="2.0", row_group_size=RG, store_schema=False)
        out.append((name, cols, sink.getvalue()))
    return out


def int_key_part(seed: int, *, sort: bool, t0: int = 0, n: int = 3 * RG) -> Dict[str, object]:
    """`value` as a group key at the ends of int64: a handful of values that repeat across vectors, row groups and
    parts.  Sorted parts hold runs of 300 equal keys (a run crosses vectors and row-group boundaries: the per-lane
    last-key cache of the hash path); unsorted parts draw every row."""
    keys = np.array([I64_MIN, I64_MIN + 1, -1, 0, 1, I64_MAX - 1, I64_MAX, 1 << 53, -(1 << 32)], dtype=np.int64)
    cols = int_part(INT_CHUNKS[:n // RG], seed, sort=sort, t0=t0)
    rng = np.random.default_rng(seed + 3)
    cols["value"] = keys[(np.arange(n) // 300 + seed) % len(keys)] if sort else keys[rng.integers(0, len(keys), n)]
    return cols


def hash_key_part(seed: int, *, t0: int = 0, n: int = 3 * RG) -> Dict[str, object]:
    """Dictionary keys for the hash table's packed key words: labels.c / labels.d with 2^12 - 1 and 2^12 values
    (12 and 13 bits of code with NULL as code 0), and labels.e .. labels.i with 9000 values each (14 bits: five keys
    cross the first 64-bit word).  Every key has its top id and a few NULLs."""
    cols = int_part(INT_CHUNKS[:n // RG], seed, sort=False, t0=t0)
    rng = np.random.default_rng(seed + 5)
    for name, card in (("c", 4095), ("d", 4096), ("e", 9000), ("f", 9000), ("g", 9000), ("h", 9000), ("i", 9000)):
        idx = rng.integers(0, card, n).astype(np.int32)
        idx[rng.choice(n, 8, replace=False)] = card - 1
        idx[rng.choice(n, 8, replace=False)] = -1
        cols[f"labels.{name}"] = (idx, label_values(card))
    return cols


def physical(cols: Dict[str, object]) -> Dict[str, np.ndarray]:
    """The columns of a part as the reference reads them: dictionary columns decoded to strings; a nullable numeric
    column (an Arrow array with a validity bitmap) as its raw slots, NULL = 0 / +0.0, with its validity under
    `<name>#valid`."""
    import pyarrow as pa
    out = {}
    for name, v in cols.items():
        if isinstance(v, tuple):
            idx, dictionary = v
            d = np.asarray(dictionary, dtype=object)
            out[name] = np.where(np.asarray(idx) < 0, None, d[np.maximum(np.asarray(idx), 0)])
        elif isinstance(v, pa.Array):
            out[name] = v.fill_null(0).to_numpy(zero_copy_only=False)
            if v.null_count:
                out[name + "#valid"] = v.is_valid().to_numpy(zero_copy_only=False)
        else:
            out[name] = np.asarray(v)
    return out


# ---- the reference -----------------------------------------------------------------------------------------------
def _leaf_mask(col: np.ndarray, op: int, lit) -> np.ndarray:
    if lit is None:
        return np.zeros(len(col), bool)  # numeric leaf against NULL: nothing
    if col.dtype == object:  # dictionary strings
        valid = np.array([x is not None for x in col], bool)
        eq = np.array([x == lit for x in col], bool)
        if op == lp.OpEq:
            return eq
        if op == lp.OpNotEq:
            return valid & ~eq
        raise ValueError(f"operator {op} on a dictionary column")
    if col.dtype.kind == "f" or isinstance(lit, float):
        x, y = col.astype(np.float64), float(lit)
    else:
        x, y = col, np.int64(lit)
    with np.errstate(invalid="ignore"):
        return {lp.OpEq: x == y, lp.OpNotEq: x != y, lp.OpLt: x < y, lp.OpLtEq: x <= y, lp.OpGt: x > y,
                lp.OpGtEq: x >= y}[op]


def selection(cols: Dict[str, np.ndarray], filt) -> np.ndarray:
    n = len(cols["timestamp"])
    if filt is None:
        return np.ones(n, bool)
    if filt.Op in (lp.OpAnd, lp.OpOr):
        a, b = selection(cols, filt.Left), selection(cols, filt.Right)
        return (a & b) if filt.Op == lp.OpAnd else (a | b)
    name = filt.Left.Name()
    if name not in cols:
        raise ValueError(f"reference: no column {name}")
    m = _leaf_mask(cols[name], filt.Op, filt.Right.Value)
    return m & cols[name + "#valid"] if name + "#valid" in cols else m


def _wrap64(x: int) -> int:
    return (x + (1 << 63)) % (1 << 64) - (1 << 63)


def _aggregate(func: int, vs: np.ndarray):
    """One group's values in row order."""
    if func == lp.AggFuncCount:
        return len(vs)
    if vs.dtype.kind == "f":
        if func == lp.AggFuncSum:
            with np.errstate(over="ignore", invalid="ignore"):  # inf and NaN are results here
                s = float(np.cumsum(vs)[-1])  # sequential: cumsum adds in row order (np.sum would add pairwise)
                # the kernels add in an order the engine does not pin: a dataset must make every order agree (the
                # sorted orders put the largest magnitudes of one sign together, where an overflow would show)
                others = [float(np.cumsum(o)[-1]) for o in (vs[::-1], np.sort(vs), np.sort(vs)[::-1])] + [float(np.sum(vs))]
            assert all(same_value(o, s, lp.AggFuncSum) for o in others), f"float Sum depends on the order: {s!r} vs {others!r}"
            return s
        # Go's `if v < m` with m seeded by the first value: a NaN first value stays, a later NaN never replaces
        if math.isnan(vs[0]):
            return float(vs[0])
        return float(np.nanmin(vs) if func == lp.AggFuncMin else np.nanmax(vs))
    if func == lp.AggFuncSum:
        return _wrap64(sum(vs.tolist()))
    return int(vs.min() if func == lp.AggFuncMin else vs.max())


def _div64(x: int, y: int) -> int:
    """Go's int64 `/`: truncates toward zero and wraps (INT64_MIN / -1 = INT64_MIN); the caller handles y == 0."""
    q = abs(x) // abs(y)
    return _wrap64(-q if (x < 0) != (y < 0) else q)


def _is_float(e, cols) -> bool:
    if isinstance(e, lp.AliasExpr):
        return _is_float(e.Expr, cols)
    if isinstance(e, lp.LiteralExpr):
        return isinstance(e.Value, float)
    if isinstance(e, lp.BinaryExpr):
        return _is_float(e.Left, cols) or _is_float(e.Right, cols)
    return np.asarray(cols[e.Name()]).dtype.kind == "f"


def eval_expr(expr, cols: Dict[str, np.ndarray], *, as_float: bool = None) -> np.ndarray:
    """An arithmetic expression over the rows of `cols` (physical() columns), as Go's projection evaluates it
    (query/physicalplan/project.go:169-281):

    - int64 `+ - *` wrap modulo 2^64; `/` truncates toward zero and INT64_MIN / -1 = INT64_MIN;
    - float64 is IEEE; a divisor that is `== 0` (+0.0 or -0.0) makes the row NULL, a NaN divisor gives NaN;
    - an int64 zero divisor makes the row NULL; a NULL produced here, like a NULL input, is read by everything
      downstream as its raw slot, 0 or +0.0 (validity is ignored, the reducers read Int64Values / Float64Values);
    - an int literal in an expression over float64 becomes a double, rounded to nearest.  Go would panic on that
      type assertion; taking the literal as a double is this engine's extension.

    Plain Python ints for int64 (wrapped explicitly) and numpy for float64; nothing from the engine or the oracle."""
    if as_float is None:
        as_float = _is_float(expr, cols)
    if isinstance(expr, lp.AliasExpr):
        return eval_expr(expr.Expr, cols, as_float=as_float)
    n = len(cols["timestamp"])
    if isinstance(expr, lp.LiteralExpr):
        v = expr.Value
        return np.full(n, float(v), np.float64) if as_float else np.full(n, int(v), np.int64)
    if not isinstance(expr, lp.BinaryExpr):
        v = np.asarray(cols[expr.Name()])
        return v.astype(np.float64) if as_float else v.astype(np.int64)
    a = eval_expr(expr.Left, cols, as_float=as_float)
    b = eval_expr(expr.Right, cols, as_float=as_float)
    op = expr.Op
    if as_float:
        with np.errstate(all="ignore"):
            if op == lp.OpAdd:
                return a + b
            if op == lp.OpSub:
                return a - b
            if op == lp.OpMul:
                return a * b
            zero = b == 0.0
            return np.where(zero, 0.0, a / np.where(zero, 1.0, b))
    x, y = a.tolist(), b.tolist()
    if op == lp.OpAdd:
        out = [_wrap64(p + q) for p, q in zip(x, y)]
    elif op == lp.OpSub:
        out = [_wrap64(p - q) for p, q in zip(x, y)]
    elif op == lp.OpMul:
        out = [_wrap64(p * q) for p, q in zip(x, y)]
    else:
        out = [0 if q == 0 else _div64(p, q) for p, q in zip(x, y)]
    return np.array(out, dtype=np.int64)


def _key_name(k) -> str:
    return k if isinstance(k, str) else k.Name()


def _key_values(k, cols) -> List[object]:
    """A group key per row: dictionary strings (None for NULL), int64 columns and computed keys as ints (NULL groups
    with 0, dynparquet/hashed.go:254-262: the raw slot is 0)."""
    if isinstance(k, str) and np.asarray(cols[k]).dtype == object:
        return list(cols[k])
    return eval_expr(lp.Col(k) if isinstance(k, str) else k, cols).tolist()


def reference(parts: Sequence[Dict[str, np.ndarray]], filt, keys: Sequence, aggs: Sequence[lp.AggregationFunction]):
    """Aggregate plans: {key tuple: tuple of aggregate values}.  `parts`: physical() of every part, in insertion
    order.  A key is a column name or an expression (computed key, named by its alias); an aggregate's input is a
    column or an expression (eval_expr).  Keys are compared by value."""
    masks = [selection(cols, filt) for cols in parts]
    n = sum(int(m.sum()) for m in masks)
    if n == 0:
        return {}
    sel = [{c: np.asarray(v)[m] for c, v in cols.items()} for cols, m in zip(parts, masks)]
    key_rows = list(zip(*[[x for cols in sel for x in _key_values(k, cols)] for k in keys])) if keys else [()] * n
    vals = [np.concatenate([eval_expr(a.Expr, cols) for cols in sel]) for a in aggs]
    groups: Dict[tuple, List[int]] = {}
    for i, kt in enumerate(key_rows):  # rows of a group stay in row order
        groups.setdefault(kt, []).append(i)
    out = {}
    for kt, rows in groups.items():
        idx = np.array(rows, dtype=np.int64)
        out[kt] = tuple(_aggregate(a.Func, v[idx]) for a, v in zip(aggs, vals))
    return out


def post_project(result: dict, names: Sequence[str], exprs: Sequence[lp.Expr]) -> dict:
    """A post-aggregate projection over a reference result ({key: values in the order of `names`}): each expression
    over the named result columns, with eval_expr's rules; a row whose division had a zero divisor is None (NULL)."""
    keys = list(result)
    cols = {nm: np.array([result[k][i] for k in keys]) for i, nm in enumerate(names)}
    cols["timestamp"] = np.zeros(len(keys), np.int64)  # eval_expr's row count
    out = {k: [] for k in keys}
    for e in exprs:
        v = eval_expr(e, cols).tolist()
        nulls = _zero_divisor_rows(e, cols)
        for i, k in enumerate(keys):
            out[k].append(None if nulls[i] else v[i])
    return {k: tuple(v) for k, v in out.items()}


def _zero_divisor_rows(e, cols) -> np.ndarray:
    """Rows that the outermost division of `e` makes NULL."""
    n = len(cols["timestamp"])
    if isinstance(e, lp.AliasExpr):
        return _zero_divisor_rows(e.Expr, cols)
    if isinstance(e, lp.BinaryExpr) and e.Op == lp.OpDiv:
        return eval_expr(e.Right, cols, as_float=_is_float(e, cols)) == 0
    return np.zeros(n, bool)


def reference_rows(parts: Sequence[Dict[str, np.ndarray]], filt, names: Sequence[str]) -> List[tuple]:
    """Filter-only plans: the selected rows in insertion order."""
    out = []
    for cols in parts:
        sel = np.flatnonzero(selection(cols, filt))
        out.extend(zip(*[[x.item() for x in cols[n][sel]] for n in names]))
    return out


# ---- plans -------------------------------------------------------------------------------------------------------
KEYS = ["labels.a", "labels.b"]
V, T, F = "value", "timestamp", "floatvalue"
AGG_INT = [lp.Sum(lp.Col(V)), lp.Min(lp.Col(V)), lp.Max(lp.Col(V)), lp.Count(lp.Col(V))]
AGG_FLOAT = [lp.Sum(lp.Col(F)), lp.Min(lp.Col(F)), lp.Max(lp.Col(F)), lp.Count(lp.Col(F))]
AGG_FLOAT_SUM = [lp.Sum(lp.Col(F)), lp.Count(lp.Col(F))]


def int_edge_filters(n_rows: int) -> List[lp.Expr]:
    """Case 1: every operator against the ends of int64 and the chunk bounds (`value`), and against the ends of int64
    and of the table (`timestamp`, 0 .. n_rows - 1)."""
    out = [leaf(V, op, x) for op in OPS for x in sorted(set(EDGE_LITERALS + chunk_literals()))]
    out += [leaf(T, op, x) for op in OPS for x in sorted(set(EDGE_LITERALS + [n_rows - 1, n_rows, RG]))]
    return out


def fused_filters() -> List[lp.Expr]:
    """Case 2: conjunctions the host fuses into one range per column (full, empty, one value wide), three leaves on one
    column, and two columns with two leaves each (beyond the sorted-run kernel's two range leaves when not fused)."""
    v = lp.Col(V)
    a = (1 << 53) - 3
    return [
        lp.And(v.GtEq(lp.Literal(I64_MIN)), v.LtEq(lp.Literal(I64_MAX))),
        lp.And(v.Gt(lp.Literal(I64_MAX)), v.GtEq(lp.Literal(0))),
        lp.And(v.Lt(lp.Literal(I64_MIN)), v.LtEq(lp.Literal(I64_MAX))),
        lp.And(v.GtEq(lp.Literal(a)), v.Lt(lp.Literal(a))),
        lp.And(v.Gt(lp.Literal(a)), v.Lt(lp.Literal(a + 2))),
        lp.And(v.Gt(lp.Literal(I64_MAX - 2)), v.Lt(lp.Literal(I64_MAX))),
        lp.And(v.Gt(lp.Literal(I64_MIN)), v.Lt(lp.Literal(I64_MIN + 2))),
        lp.And(v.GtEq(lp.Literal(-1)), v.LtEq(lp.Literal(0))),
        lp.And(lp.And(v.Gt(lp.Literal(-7)), v.LtEq(lp.Literal(200))), v.Lt(lp.Literal(I64_MAX))),
        lp.And(lp.And(v.GtEq(lp.Literal(I64_MIN)), v.Lt(lp.Literal(I64_MIN + 40_000))), v.Gt(lp.Literal(I64_MIN))),
        lp.And(lp.And(v.GtEq(lp.Literal(0)), v.LtEq(lp.Literal(I64_MAX))),
               lp.And(lp.Col(T).GtEq(lp.Literal(RG // 2)), lp.Col(T).Lt(lp.Literal(9 * RG + 5)))),
        lp.And(lp.And(v.Gt(lp.Literal(I64_MIN)), v.Lt(lp.Literal(I64_MAX))),
               lp.And(lp.Col(T).Gt(lp.Literal(-1)), lp.Col(T).LtEq(lp.Literal(I64_MAX)))),
    ]


def int_float_filters() -> List[lp.Expr]:
    """Case 3: the int64 column against float literals: fractions, signed zeros, 2^53 and 2^53 + 2 against values
    that round, literals beyond int64, infinities and NaN."""
    lits = [2.5, -0.5, 0.0, -0.0, float(1 << 53), float((1 << 53) + 2), 9.3e18, -9.3e18, INF, -INF, NAN]
    return [leaf(V, op, x) for op in OPS for x in lits]


def float_filters() -> List[lp.Expr]:
    """Case 4: the float64 column against its specials, and an int literal above 2^53 (compared as a double)."""
    lits = [NAN, INF, -INF, 0.0, -0.0, DENORM_MIN, DBL_MAX, 0.5, (1 << 53) + 1]
    return [leaf(F, op, x) for op in OPS for x in lits]


# ---- expression plans (aggregate inputs, computed keys) ---------------------------------------------------------------
def _c(name):
    return lp.Col(name)


def _l(v):
    return lp.Literal(v)


def _all4(e) -> List[lp.AggregationFunction]:
    return [lp.Sum(e), lp.Min(e), lp.Max(e), lp.Count(e)]


def int_expr_inputs() -> List[lp.Expr]:
    """Int64 aggregate inputs: wrapping + - *, division over DIVISORS (timestamp) and by 0, literals on the left, and
    programs of depth 3."""
    v, t = _c(V), _c(T)
    return [lp.Add(v, t), lp.Sub(v, t), lp.Mul(v, t), lp.Mul(v, v), lp.Div(v, t), lp.Sub(_l(I64_MIN), v),
            lp.Div(_l(7), v), lp.Div(v, _l(0)), lp.Div(v, _l(-1)), lp.Mul(lp.Sub(v, t), lp.Add(v, _l(1))),
            lp.Div(v, lp.Sub(t, _l(3)))]


def many_int_aggs() -> List[lp.AggregationFunction]:
    """Eight expression aggregates in one plan: 42 program ops, 47 of kMaxProg = 48 with the 5-op key bucket(1000)
    behind them."""
    v, t = _c(V), _c(T)
    return [lp.Sum(lp.Mul(lp.Sub(v, t), lp.Add(v, _l(1)))), lp.Min(lp.Div(v, lp.Sub(t, _l(3)))),
            lp.Max(lp.Mul(lp.Add(v, t), lp.Sub(t, _l(2)))), lp.Sum(lp.Div(lp.Add(v, _l(5)), lp.Sub(t, _l(1)))),
            lp.Min(lp.Sub(lp.Mul(v, _l(3)), t)), lp.Max(lp.Add(lp.Div(v, t), t)),
            lp.Sum(lp.Sub(lp.Sub(v, _l(I64_MAX)), t)), lp.Count(v)]


def expr_filters() -> List[lp.Expr]:
    """No filter, a conjunction, and an OR (the general filter program)."""
    return [None, lp.And(leaf(V, lp.OpGt, I64_MIN), leaf("labels.a", lp.OpNotEq, "v000001")),
            lp.Or(leaf(V, lp.OpLt, -1), leaf(T, lp.OpEq, 0))]


def float_expr_aggs() -> List[List[lp.AggregationFunction]]:
    """Float64 aggregate inputs over floatvalue (with NULL rows).  Inputs whose Sum would depend on the summation
    order (a big addend, reciprocals) take Min / Max / Count only."""
    f = _c(F)
    big = (1 << 53) + 1  # an int literal: a double, 2^53
    return [_all4(lp.Mul(f, _l(2))), [lp.Min(lp.Add(f, _l(big))), lp.Max(lp.Add(f, _l(big))), lp.Count(f)],
            _all4(lp.Div(f, _l(0.0))), _all4(lp.Div(f, _l(-0.0))), _all4(lp.Div(f, _l(0))), _all4(lp.Sub(f, f)),
            _all4(lp.Div(f, f)), [lp.Min(lp.Div(_l(1.0), f)), lp.Max(lp.Div(_l(1.0), f)), lp.Count(f)]]


def bucket(k: int, name: str = "bucket") -> lp.Expr:
    """The time bucket of Parca's Range query: (timestamp / k) * k."""
    return lp.Mul(lp.Div(_c(T), _l(k)), _l(k)).Alias(name)


BUCKET_WIDTHS = [1, 7, 1000, -1000, I64_MAX, I64_MIN]


def computed_key_sets() -> List[list]:
    v, t = _c(V), _c(T)
    return [[bucket(k)] for k in BUCKET_WIDTHS] + [
        [lp.Mul(v, _l(3)).Alias("v3")], [lp.Sub(v, t).Alias("vt")], [lp.Div(v, t).Alias("vdt")],
        ["labels.a", bucket(1000), "timestamp", lp.Div(v, t).Alias("vdt")]]


_FIVE = ["labels.e", "labels.f", "labels.g", "labels.h", "labels.i"]
# hash_key_part's keys: 12 + 13 bits of code in one word; 5 x 14 bits across two words; and those two words with
# two int64 and two computed keys: six words, kMaxKeyWords
HASH_KEY_SETS = [["labels.c", "labels.d"], _FIVE, ["labels.d"] + _FIVE,
                 _FIVE + [V, T, bucket(1000), lp.Div(_c(V), _c(T)).Alias("vdt")]]


def oracle_groups_exactly(keys, cols) -> bool:
    """The oracle keys groups by a 64-bit hash only, as Go does (aggregate.go:411): an int64 key hashes as its value
    (hashed.go:254-262) and hashCombine is not injective over two of them, so small int64 keys in two columns merge
    distinct groups there.  The engine compares packed keys exactly.  With at most one int64 key the combined hash is
    injective in it and the oracle's groups are the exact ones."""
    return sum(1 for k in keys if not isinstance(k, str) or np.asarray(cols[k]).dtype != object) <= 1


def has_nan_minmax(aggs) -> bool:
    """Plans whose Min / Max over floatvalue may see NaN (the oracle's merge order decides their NaN at 4 threads)."""
    return any(a.Func in (lp.AggFuncMin, lp.AggFuncMax) and a.Expr.Name() == F for a in aggs)


# ---- comparison --------------------------------------------------------------------------------------------------
def result_map(batches, keys: Sequence[str], aggs: Sequence[lp.AggregationFunction]):
    """Engine / oracle records as {key tuple: tuple of aggregate values}."""
    import pyarrow as pa
    names = [a.Name() for a in aggs]
    out = {}
    for b in batches:
        cols = []
        for n in list(keys) + names:
            c = b.column(b.schema.get_field_index(n))
            if pa.types.is_dictionary(c.type):
                c = c.dictionary_decode()
            cols.append([x.decode() if isinstance(x, bytes) else x for x in c.to_pylist()])
        for r in zip(*cols):
            k = tuple(r[:len(keys)])
            assert k not in out, f"group {k} twice"
            out[k] = tuple(r[len(keys):])
    return out


def _bits(x: float) -> int:
    return struct.unpack("<q", struct.pack("<d", x))[0]


def same_value(got, exp, func: int) -> bool:
    """Integers exactly; floats bit for bit, except that all NaNs are equal and, for Min / Max, -0.0 == +0.0."""
    if isinstance(exp, float) or isinstance(got, float):
        if not (isinstance(exp, float) and isinstance(got, float)):
            return False
        if math.isnan(exp) or math.isnan(got):
            return math.isnan(exp) and math.isnan(got)
        if func in (lp.AggFuncMin, lp.AggFuncMax) and exp == 0.0:
            return got == 0.0
        return _bits(got) == _bits(exp)
    if isinstance(exp, int) and isinstance(got, int):
        return got == exp
    return got == exp  # strings (filter-only rows)


def assert_same_result(got: dict, exp: dict, aggs: Sequence[lp.AggregationFunction], what: str = "") -> None:
    # (sorted by repr: a NULL key is None, which does not order against strings)
    assert set(got) == set(exp), f"{what}: groups differ: only engine {sorted(set(got) - set(exp), key=repr)[:5]}, only reference {sorted(set(exp) - set(got), key=repr)[:5]}"
    for k, ev in exp.items():
        gv = got[k]
        for a, g, e in zip(aggs, gv, ev):
            assert same_value(g, e, a.Func), f"{what}: group {k} {a.Name()}: got {g!r}, expected {e!r}"


def record_rows(batches, names: Sequence[str]) -> List[tuple]:
    """Rows of filter-only records in record order (empty records carry no columns)."""
    return [r for b in batches if b.num_rows for r in zip(*[b.column(b.schema.get_field_index(n)).to_pylist() for n in names])]


def assert_same_rows(got: List[tuple], exp: List[tuple], what: str = "") -> None:
    assert len(got) == len(exp), f"{what}: {len(got)} rows, expected {len(exp)}"
    for i, (g, e) in enumerate(zip(got, exp)):
        assert all(same_value(x, y, 0) for x, y in zip(g, e)), f"{what}: row {i}: got {g!r}, expected {e!r}"
