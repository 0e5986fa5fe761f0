"""Upload cost of LZ4_RAW-compressed parts (PLAIN int64 values inflated on the device at upload, everything else on
the host at the page walk) against their uncompressed twin.

On the benchmark's shape (bench_data.part_columns: sorted parts of 4 Mi rows, 1 Mi-row row groups, 16 Mi rows in all,
4 label columns) with every column LZ4_RAW next to the same rows uncompressed, and the benchmark's plan
(timestamp in the middle half of the range, Sum(value) and Count(value) by labels.l00, labels.l01), it reports
  put_ms                  fgpu_part_put_parquet of every part (eager: the whole part goes to the device)
  put_first_execute_ms    the same, then one Execute
  borrowed_first_*        the first Execute over freshly borrowed parts: its wall time and h2d_bytes
  steady_execute_ms       the median of further Executes through the C ABI (result conversion not included), and
  steady_device_ms        their fgpu_stats total_device_ms
  lz4_pages               per part: the pages k_lz4_pages inflates (one warp each) and their inflated bytes
  decode_us               k_lz4_pages device time (torch.profiler) in an eager put of the LZ4_RAW parts, a run of its own
with a host clock around calls that end in a device synchronise.  Prints one JSON line per measurement, then one with
all of them and the card's name and power limit, which --out also writes to a file.

    python scripts/lz4_upload.py [--parts N] [--reps K] [--data-page-size BYTES] [--out FILE]
"""
import argparse
import ctypes as C
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import bench_data as bd  # noqa: E402
from frostdb_b200 import _lib  # noqa: E402
from frostdb_b200 import dynparquet as dp  # noqa: E402
from frostdb_b200 import logicalplan as lp  # noqa: E402
from frostdb_b200 import query  # noqa: E402
from frostdb_b200.physicalplan import GPUScan  # noqa: E402
from frostdb_b200.store import ColumnStore  # noqa: E402
from plain_strings_upload import card  # noqa: E402

N_LABELS = 4
KEYS = [lp.Col("labels.l00"), lp.Col("labels.l01")]
AGGS = [lp.Sum(lp.Col("value")), lp.Count(lp.Col("value"))]


def schema(lz4: bool) -> dp.Schema:
    c = "LZ4_RAW" if lz4 else "NONE"
    s = dp.Schema(name="lz4", columns=[dp.ColumnDefinition("example_type", dp.TYPE_STRING, rle_dictionary=True, compression=c),
                                        dp.ColumnDefinition("labels", dp.TYPE_STRING, nullable=True, dynamic=True, rle_dictionary=True,
                                                            compression=c),
                                        dp.ColumnDefinition("stacktrace", dp.TYPE_STRING, rle_dictionary=True, compression=c),
                                        dp.ColumnDefinition("timestamp", dp.TYPE_INT64, compression=c),
                                        dp.ColumnDefinition("value", dp.TYPE_INT64, compression=c)],
                  sorting_columns=[dp.SortingColumn("example_type"), dp.SortingColumn("labels", nulls_first=True),
                                   dp.SortingColumn("timestamp"), dp.SortingColumn("stacktrace", nulls_first=True)])
    return s


def parts(n_parts: int, lz4: bool, page: int):
    cards = bd.cardinalities(N_LABELS)
    out = []
    for k in range(n_parts):
        cols = bd.part_columns(k * bd.PART_ROWS, bd.PART_ROWS, N_LABELS, cards)
        out.append(np.frombuffer(dp.write_part(schema(lz4), cols, sort=False, row_group_size=bd.RG_ROWS, data_page_size=page), dtype=np.uint8))
    return out


def plan_filter(n_rows: int):
    t = lp.Col("timestamp")
    return lp.And(t.GtEq(lp.Literal(bd.T0 + n_rows // 4)), t.Lt(lp.Literal(bd.T0 + 3 * n_rows // 4)))


def execute(db, table: str, filt):
    out = []
    query.NewEngine(None, db.TableProvider()).ScanTable(table).Filter(filt).Aggregate(AGGS, KEYS).Execute(None, lambda c, r: out.append(r))
    return sorted(tuple(r) for b in out if b.num_rows for r in zip(*[b.column(i).to_pylist() for i in range(b.num_columns)]))


def stats_execute(cs, table: str, filt) -> dict:
    eng, lib = cs.engine, _lib.load()
    q, keep = GPUScan(eng, table, filt, _lib.PLAN_AGGREGATE, KEYS, AGGS).prepare()
    res = C.c_void_p()
    try:
        _lib.check(lib.fgpu_query_execute(eng.handle, q, eng.table_watermark(table), C.byref(res)))
        st = eng.stats(res)
        lib.fgpu_result_free(res)
    finally:
        lib.fgpu_query_free(q)
    return st


def decode_us(cs, db, bufs) -> dict:
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    us = {}
    for rep in ("warm", "measured"):
        name = f"lz4_prof_{rep}"
        db.Table(name, schema(True))
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for b in bufs:
                cs.engine.put_parquet(name, b)
        cs.engine.drop_table(name)
        db.tables.pop(name, None)
        us = {}
        for e in prof.events():
            if e.device_type.name == "CUDA" and "k_lz4_pages" in e.name:
                us["k_lz4_pages"] = us.get("k_lz4_pages", 0.0) + e.device_time
    return {k: round(v, 1) for k, v in sorted(us.items())}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--parts", type=int, default=4)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--data-page-size", type=int, default=1 << 20, help="pyarrow's data_page_size (pages per column chunk)")
    ap.add_argument("--out", default=None, help="also write the result JSON to this file")
    args = ap.parse_args()
    n_rows = args.parts * bd.PART_ROWS
    filt = plan_filter(n_rows)
    inputs = {"lz4": parts(args.parts, True, args.data_page_size), "plain": parts(args.parts, False, args.data_page_size)}
    pages = {}
    for col in ("timestamp", "value"):
        d = _lib.describe_parquet(inputs["lz4"][0].tobytes())
        cs_ = [rg["columns"][col] for rg in d["row_groups"]]
        pages[col] = {"device_pages": sum(c["lz4_device_pages"] for c in cs_), "inflated_bytes": sum(c["stored_bytes"] for c in cs_)}
    print(json.dumps({"lz4_pages": pages}), flush=True)
    cs = ColumnStore(0)
    db = cs.DB(None, "lz4_upload")
    results, answers = [], {}
    for rep, bufs in inputs.items():
        r = {"rep": rep, "file_bytes": int(sum(b.nbytes for b in bufs))}
        name = f"lz4_{rep}_eager"
        db.Table(name, schema(rep == "lz4"))
        t0 = time.perf_counter()
        for b in bufs:
            cs.engine.put_parquet(name, b)
        t1 = time.perf_counter()
        answers[rep] = execute(db, name, filt)
        t2 = time.perf_counter()
        r["put_ms"], r["put_first_execute_ms"] = round((t1 - t0) * 1e3, 2), round((t2 - t0) * 1e3, 2)
        steady, device = [], []
        for _ in range(args.reps):
            a = time.perf_counter()
            st = stats_execute(cs, name, filt)
            steady.append(time.perf_counter() - a)
            device.append(float(st["total_device_ms"]))
        r["steady_execute_ms"] = round(statistics.median(steady) * 1e3, 3)
        r["steady_device_ms"] = round(statistics.median(device), 3)
        cs.engine.drop_table(name)
        db.tables.pop(name, None)
        name = f"lz4_{rep}_borrowed"
        db.Table(name, schema(rep == "lz4"))
        for b in bufs:
            cs.engine.put_parquet(name, b, borrow=True)
        a = time.perf_counter()
        st = stats_execute(cs, name, filt)
        r["borrowed_first_execute_ms"] = round((time.perf_counter() - a) * 1e3, 2)
        r["borrowed_first_h2d_bytes"] = int(st["h2d_bytes"])
        cs.engine.drop_table(name)
        db.tables.pop(name, None)
        results.append(r)
        print(json.dumps(r), flush=True)
    assert answers["lz4"] == answers["plain"], "the LZ4_RAW parts answer differently from their uncompressed twins"
    try:
        dec = decode_us(cs, db, inputs["lz4"])
    except Exception as e:  # (the upload numbers are still reported)
        dec = {"error": repr(e)}
    print(json.dumps({"decode_us": dec}), flush=True)
    cs.Close()
    out = {"rows": n_rows, "data_page_size": args.data_page_size, **card(), "results": results, "lz4_pages": pages, "decode_us": dec}
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
