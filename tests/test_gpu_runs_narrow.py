"""Frame-of-reference images of the sorted-run kernel (ensure_narrow, k_runs_tma): int64 chunks whose range fits 8, 16
or 32 bits are staged as value - min in that width and widened on the device.  Chunk ranges at the width boundaries,
negative and extreme bases, sums that wrap, ranges and Min / Max on narrowed columns, row groups of different widths in
one launch and files without statistics, each against the oracle and the general scan kernel (run3)."""
import numpy as np
import pytest

from frostdb_b200 import logicalplan as lp
from tests.test_gpu_runs import AGGS, KEYS, pair, run3, scan_stats  # noqa: F401  (pair: fixture)
from tests.util import label_values

pytestmark = pytest.mark.gpu

I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
RG = 6_000


def part_with_chunks(chunks, seed, t0=0):
    """One part whose row group k holds RG rows with `value` in [lo_k, hi_k], both ends present.  The label and timestamp
    columns are generated in the order compaction writes them, so row group k is rows [k * RG, (k + 1) * RG)."""
    n = RG * len(chunks)
    rng = np.random.default_rng(seed)
    g = np.sort(rng.integers(0, 5 * 11, n))  # sorted (a, b): long runs
    value = np.empty(n, np.int64)
    for k, (lo, hi) in enumerate(chunks):
        v = lo + (rng.integers(0, 1 << 62, RG, dtype=np.int64).astype(object) % (hi - lo + 1))
        v[rng.integers(0, RG)] = lo
        v[rng.integers(0, RG)] = hi
        value[k * RG:(k + 1) * RG] = np.array([int(x) for x in v], dtype=np.int64)
    return {
        "example_type": (np.zeros(n, np.int32), ["cpu"]),
        "stacktrace": (rng.integers(0, 7, n).astype(np.int32), [f"stack{i:02d}" for i in range(7)]),
        "timestamp": t0 + np.arange(n, dtype=np.int64),
        "value": value,
        "labels.a": ((g // 11).astype(np.int32), label_values(5)),
        "labels.b": ((g % 11).astype(np.int32), label_values(11)),
    }


# (lo, hi) per row group: ranges of exactly 2^8 - 1 / 2^8, 2^16 - 1 / 2^16, 2^32 - 1 / 2^32, negative bases
BOUNDARY = [(-7, 248), (1000, 1256), (-(1 << 40), -(1 << 40) + 65535), (3, 65539), (-(1 << 31), (1 << 31) - 1), (17, 17 + (1 << 32))]
# the ends of int64: sums wrap (modulo 2^64, as Go's int64 does); one chunk needs all 64 bits
EXTREMES = [(I64_MAX - 200, I64_MAX), (I64_MIN, I64_MIN + 70_000), (I64_MIN, I64_MAX), (-1, 0), (I64_MAX - (1 << 32) + 1, I64_MAX)]


def value_filters(chunks):
    """Range leaves on `value` with bounds outside, at and inside the chunks' ranges."""
    v = lp.Col("value")
    out = []
    for lo, hi in chunks[:4]:
        mid = lo + (hi - lo) // 2
        out += [v.GtEq(lp.Literal(lo)), v.Gt(lp.Literal(lo)), v.LtEq(lp.Literal(hi)), v.Lt(lp.Literal(hi)),
                lp.And(v.GtEq(lp.Literal(max(lo - 1, I64_MIN))), v.LtEq(lp.Literal(mid))), lp.And(v.Gt(lp.Literal(mid)), v.Lt(lp.Literal(min(hi + 1, I64_MAX))))]
    return out


def check(p, chunks):
    v, ts = lp.Col("value"), lp.Col("timestamp")
    run3(p, lambda q: q.Aggregate(AGGS, KEYS))
    run3(p, lambda q: q.Aggregate([lp.Sum(v), lp.Min(v), lp.Max(v), lp.Count(v)], KEYS))
    run3(p, lambda q: q.Aggregate([lp.Min(v), lp.Max(v)], []))
    tf = lp.And(ts.GtEq(lp.Literal(RG // 2)), ts.Lt(lp.Literal(len(chunks) * RG - 77)))  # boundary row groups: per-row test
    run3(p, lambda q: q.Filter(tf).Aggregate([lp.Sum(v), lp.Min(v), lp.Max(v), lp.Count(v)], KEYS))
    for f in value_filters(chunks):
        try:
            run3(p, lambda q: q.Filter(f).Aggregate(AGGS, KEYS))
            run3(p, lambda q: q.Filter(lp.And(f, tf)).Aggregate([lp.Min(v), lp.Max(v), lp.Sum(ts)], [lp.Col("labels.a")]))
        except AssertionError as e:
            raise AssertionError(f"filter {f.Name()}: {e}") from e


@pytest.mark.parametrize("stats", [True, False])
def test_chunk_ranges_at_the_width_boundaries(pair, stats):
    p = pair("narrow_bounds")
    p.insert(part_with_chunks(BOUNDARY[:3], 1), row_group_size=RG, write_statistics=stats)
    p.insert(part_with_chunks(BOUNDARY[3:], 2, t0=3 * RG), row_group_size=RG, write_statistics=stats)
    check(p, BOUNDARY)
    st = scan_stats(p, None, AGGS, KEYS)
    assert st["row_groups_runs"] == st["row_groups"] == 6  # one launch, row groups of 8, 16, 32 and 64 bits
    assert st["algorithmic_bytes"] < 6 * RG * 8  # narrowed chunks count their staged width


def test_int64_extremes_and_wrapping_sums(pair):
    p = pair("narrow_extremes")
    p.insert(part_with_chunks(EXTREMES, 3), row_group_size=RG)
    check(p, EXTREMES)
