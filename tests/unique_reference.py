"""A plain reference for the Unique(int64) aggregate: Python ints over rows, no engine or oracle code.

The rule (physicalplan/aggregate.go:677-730): a group's Unique is its value when every row of the group is non-NULL and
all rows hold the same value, and NULL otherwise, a group with any NULL row included.  The final stage runs the same
function over the partial results, so a NULL partial makes the result NULL and the answer does not depend on how the
rows were split.
"""
from __future__ import annotations

from typing import Callable, Dict, List, Optional, Sequence

_NULL = object()  # a group that has met a NULL row, or two different values


def unique(values: Sequence[Optional[int]]) -> Optional[int]:
    """Unique over one group's values (None = NULL); an empty sequence has no group and no answer."""
    if not values:
        raise ValueError("a group has at least one row")
    first = values[0]
    if first is None or any(v != first for v in values):
        return None
    return int(first)


def grouped(keys: Sequence[tuple], values: Sequence[Optional[int]]) -> Dict[tuple, Optional[int]]:
    """Unique per group: keys[i] is row i's group, values[i] its value."""
    out: Dict[tuple, object] = {}
    for k, v in zip(keys, values):
        cur = out.get(k, v if v is not None else _NULL)
        out[k] = _NULL if (v is None or cur is _NULL or cur != v) else cur
    return {k: (None if v is _NULL else int(v)) for k, v in out.items()}


def rows(parts: Sequence[Dict[str, list]], keys: Sequence[Callable[[Dict[str, list], int], object]],
         columns: Sequence[str], selected: Optional[Callable[[Dict[str, list], int], bool]] = None) -> List[tuple]:
    """Result rows (key values..., Unique of each of `columns`...) over the parts' rows that `selected` keeps, sorted
    with NULLs last.  A part is column name -> values (None = NULL); a key is a function of (part, row)."""
    group_keys: List[tuple] = []
    values: Dict[str, List[Optional[int]]] = {c: [] for c in columns}
    for part in parts:
        n = len(next(iter(part.values())))
        for i in range(n):
            if selected is not None and not selected(part, i):
                continue
            group_keys.append(tuple(k(part, i) for k in keys))
            for c in columns:
                values[c].append(part[c][i])
    per_col = [grouped(group_keys, values[c]) for c in columns]
    out = [k + tuple(g[k] for g in per_col) for k in dict.fromkeys(group_keys)]
    return sorted(out, key=lambda r: tuple((x is None, x) for x in r))
