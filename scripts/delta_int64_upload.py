"""Upload cost of DELTA_BINARY_PACKED int64 columns (decoded on the device at upload) against their PLAIN twin.

On the benchmark's shape (bench_data.part_columns: sorted parts of 4 Mi rows, 1 Mi-row row groups, 16 Mi rows in all,
4 label columns) with `timestamp` and `value` DELTA_BINARY_PACKED next to the same rows PLAIN, and the benchmark's plan
(timestamp in the middle half of the range, Sum(value) and Count(value) by labels.l00, labels.l01), it reports
  put_ms                  fgpu_part_put_parquet of every part (eager: the whole part goes to the device)
  put_first_execute_ms    the same, then one Execute
  borrowed_first_*        the first Execute over freshly borrowed parts: its wall time and h2d_bytes
  steady_execute_ms       the median of further Executes through the C ABI (result conversion not included), and
  steady_device_ms        their fgpu_stats total_device_ms
  decode_us               k_dbp_* device time (torch.profiler) in an eager put of the delta parts, a run of its own
with a host clock around calls that end in a device synchronise.  Prints one JSON line per measurement, then one with
all of them and the card's name and power limit, which --out also writes to a file.

    python scripts/delta_int64_upload.py [--parts N] [--reps K] [--out FILE]
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


def schema(delta: bool) -> dp.Schema:
    s = dp.Schema(name="dbp", columns=[dp.ColumnDefinition("example_type", dp.TYPE_STRING, rle_dictionary=True),
                                        dp.ColumnDefinition("labels", dp.TYPE_STRING, nullable=True, dynamic=True, rle_dictionary=True),
                                        dp.ColumnDefinition("stacktrace", dp.TYPE_STRING, rle_dictionary=True),
                                        dp.ColumnDefinition("timestamp", dp.TYPE_INT64, delta_binary_packed=delta),
                                        dp.ColumnDefinition("value", dp.TYPE_INT64, delta_binary_packed=delta)],
                  sorting_columns=[dp.SortingColumn("example_type"), dp.SortingColumn("labels", nulls_first=True),
                                   dp.SortingColumn("timestamp"), dp.SortingColumn("stacktrace", nulls_first=True)])
    return s


def parts(n_parts: int, delta: bool):
    cards = bd.cardinalities(N_LABELS)
    out = []
    for k in range(n_parts):
        cols = bd.part_columns(k * bd.PART_ROWS, bd.PART_ROWS, N_LABELS, cards)
        out.append(np.frombuffer(dp.write_part(schema(delta), cols, sort=False, row_group_size=bd.RG_ROWS), dtype=np.uint8))
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
        name = f"dbp_prof_{rep}"
        db.Table(name, schema(True))
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for b in bufs:
                cs.engine.put_parquet(name, b)
        cs.engine.drop_table(name)
        db.tables.pop(name, None)
        us = {}
        for e in prof.events():
            if e.device_type.name == "CUDA" and "k_dbp_" in e.name:
                k = "k_dbp_" + e.name.split("k_dbp_")[1].split("(")[0].split("E")[0]
                us[k] = us.get(k, 0.0) + e.device_time
    return {k: round(v, 1) for k, v in sorted(us.items())}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--parts", type=int, default=4)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default=None, help="also write the result JSON to this file")
    args = ap.parse_args()
    n_rows = args.parts * bd.PART_ROWS
    filt = plan_filter(n_rows)
    inputs = {"delta": parts(args.parts, True), "plain": parts(args.parts, False)}
    cs = ColumnStore(0)
    db = cs.DB(None, "dbp_upload")
    results, answers = [], {}
    for rep, bufs in inputs.items():
        r = {"rep": rep, "file_bytes": int(sum(b.nbytes for b in bufs))}
        name = f"dbp_{rep}_eager"
        db.Table(name, schema(rep == "delta"))
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
        name = f"dbp_{rep}_borrowed"
        db.Table(name, schema(rep == "delta"))
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
    assert answers["delta"] == answers["plain"], "the delta parts answer differently from their PLAIN twins"
    try:
        dec = decode_us(cs, db, inputs["delta"])
    except Exception as e:  # (the upload numbers are still reported)
        dec = {"error": repr(e)}
    print(json.dumps({"decode_us": dec}), flush=True)
    cs.Close()
    out = {"rows": n_rows, **card(), "results": results, "decode_us": dec}
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
