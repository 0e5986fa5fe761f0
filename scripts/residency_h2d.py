"""Bytes copied to the device by the first Execute over borrowed parts, and what that Execute returned, for every fixture
family: the layouts of tests/plain_strings.py, tests/delta_strings.py, tests/delta_int64.py, tests/lz4_pages.py (numeric
and string) and tests/hybrid_pages.py (those it can read), an Arrow part, and bench_data parts.

Each file is put with FGPU_PUT_BORROW_PINNED into a table of its own, so nothing goes to the device until a query needs
it.  One filter-only Execute per table projects every column, so it makes the whole part resident; its filter keeps
the first 1 000 timestamps.  Per family the script prints one JSON line: the summed h2d_bytes of those Executes and a
SHA-1 digest of their rows.  A change to the upload path that keeps both keeps the bytes it moves and what the
queries read.

    python scripts/residency_h2d.py
"""
import ctypes as C
import hashlib
import io
import json
import os
import sys

import numpy as np
import pyarrow.compute as pc
import pyarrow.parquet as pq

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench_data  # noqa: E402
from frostdb_b200 import _lib  # noqa: E402
from frostdb_b200 import dynparquet as dp  # noqa: E402
from frostdb_b200 import logicalplan as lp  # noqa: E402
from frostdb_b200.physicalplan import GPUScan  # noqa: E402
from frostdb_b200.store import ColumnStore  # noqa: E402
from tests import delta_int64 as di  # noqa: E402
from tests import delta_strings as ds  # noqa: E402
from tests import hybrid_pages as hp  # noqa: E402
from tests import lz4_pages as lz  # noqa: E402
from tests import plain_strings as ps  # noqa: E402


def families():
    """name -> list of (schema, parquet bytes or Arrow record)."""
    bench_schema = dp.SampleDefinition()
    cards = bench_data.cardinalities(4)
    bench = [dp.write_part(bench_schema, bench_data.part_columns(r, 50_000, 4, cards), sort=False, row_group_size=8192)
             for r in (0, 50_000)]
    return {
        "plain_strings": [(ps.schema(), ps.file_of(n)) for n in ps.NAMES],
        "delta_strings": [(ps.schema(), ds.file_of(n, e)) for n, e in ds.CASES],
        "delta_int64": [(di.schema(di.columns(n), delta=True, nullable_value=di.LAYOUT_BY_NAME[n].nullable), di.file_of(n))
                        for n in di.NAMES],
        "lz4_pages": [(lz.schema(n, lz4=True), lz.file_of(n)) for n in lz.NAMES] +
                     [(lz.str_schema(), lz.str_file_of(n)) for n in lz.STR_NAMES],
        "hybrid_pages": [(hp.schema(), hp.file_of(l.name)) for l in hp.LAYOUTS if l.error is None],
        "arrow": [(ps.schema(), ps.record_of(n)) for n in ps.NAMES[:2]],
        "bench_data": [(bench_schema, b) for b in bench],
    }


def first_execute(store, table, names, ts0):
    """h2d_bytes and rows of one filter-only Execute projecting `names`."""
    eng, lib = store.engine, _lib.load()
    filt = lp.Col("timestamp").Lt(lp.Literal(ts0 + 1000))
    q, keep = GPUScan(eng, table, filt, _lib.PLAN_FILTER, [lp.Col(n) for n in names], []).prepare()
    res = C.c_void_p()
    try:
        _lib.check(lib.fgpu_query_execute(eng.handle, q, eng.table_watermark(table), C.byref(res)))
        h2d = eng.stats(res)["h2d_bytes"]
        rows = [r for b in eng.drain(res) if b.num_rows
                for r in zip(*[b.column(b.schema.get_field_index(n)).to_pylist() for n in names])]
        lib.fgpu_result_free(res)
    finally:
        lib.fgpu_query_free(q)
    return h2d, rows


def main():
    store = ColumnStore(0)
    db = store.DB(None, "residency_h2d")
    keep = []
    for fam, items in families().items():
        h2d, digest, n_rows = 0, hashlib.sha1(), 0
        for i, (schema, src) in enumerate(items):
            table = f"{fam}_{i}"
            db.Table(table, schema)
            if isinstance(src, bytes):
                arr = np.frombuffer(src, dtype=np.uint8)
                keep.append(arr)
                store.engine.put_parquet(table, arr, borrow=True)
                t = pq.read_table(io.BytesIO(src))
            else:
                store.engine.put_arrow(table, src)
                t = src
            names = list(t.schema.names)
            ts0 = int(pc.min(t.column("timestamp")).as_py())
            b, rows = first_execute(store, table, names, ts0)
            h2d += b
            n_rows += len(rows)
            digest.update(repr((table, sorted(rows, key=repr))).encode())
            store.engine.drop_table(table)
        print(json.dumps({"family": fam, "parts": len(items), "h2d_bytes": h2d, "rows": n_rows, "digest": digest.hexdigest()}),
              flush=True)
    store.Close()


if __name__ == "__main__":
    main()
