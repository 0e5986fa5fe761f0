"""The three ways a page's int64 values reach a chunk's dense value array on the device (copied from the file, decoded
from a DELTA_BINARY_PACKED stream, inflated from an LZ4_RAW block), interleaved in one chunk's page list and filled by
one upload: put eagerly and borrowed, Sum / Count / Min / Max of `value`, with and without a range filter on it, equal
what pyarrow reads."""
import io

import numpy as np
import pyarrow.parquet as pq
import pytest

from frostdb_b200 import logicalplan as lp
from tests import lz4_pages as lz
from tests.test_gpu_delta_int64 import V, agg, two_columns

pytestmark = pytest.mark.gpu


def _wrap(x: int) -> int:
    return (x + (1 << 63)) % (1 << 64) - (1 << 63)


@pytest.mark.parametrize("borrow", [False, True])
def test_aggregates_over_every_kind_of_page(store, borrow):
    buf, _ = lz.mixed_fills()
    vals = pq.read_table(io.BytesIO(buf)).column("value").to_pylist()
    lo, hi = sorted(vals)[len(vals) // 4], sorted(vals)[3 * len(vals) // 4]
    sch = two_columns()
    for c in sch.columns:
        c.delta_binary_packed = False
    db = store.DB(None, "value_pages")
    table = f"value_pages_{int(borrow)}"
    if table in db.tables:
        store.engine.drop_table(table)
    db.Table(table, sch)
    arr = np.frombuffer(buf, dtype=np.uint8)  # (a borrowed part's bytes stay alive until it is dropped)
    try:
        store.engine.put_parquet(table, arr, borrow=borrow)
        aggs = [lp.Sum(V), lp.Count(V), lp.Min(V), lp.Max(V)]
        for filt, keep in ((None, vals), (lp.And(V.GtEq(lp.Literal(lo)), V.Lt(lp.Literal(hi))), [v for v in vals if lo <= v < hi])):
            assert keep
            assert agg(db, table, filt, [], aggs) == {(): (_wrap(sum(keep)), len(keep), min(keep), max(keep))}, filt
    finally:
        store.engine.drop_table(table)
        db.tables.pop(table, None)
