"""Upload cost of PLAIN, DELTA_LENGTH_BYTE_ARRAY and DELTA_BYTE_ARRAY string columns (interned on the device at put)
against the same column as RLE_DICTIONARY and the same rows as an Arrow part (interned on the host, row by row).

For 4 Mi-row parts whose string column `s` has 16, 64 Ki and 4 Mi distinct values, and each representation, it times
  put + first Execute   a fresh table: fgpu_part_put_* (the whole part goes to the device), then one Execute
  steady Execute        the median of further Executes of the same plan
with a host clock around calls that end in a device synchronise.  The plan counts the rows whose `s` differs from a
literal, so it reads every value of `s`.  Prints one JSON line per measurement, then one with all of them and the
card's name and power limit, which --out also writes to a file.

It also reports the device time of k_str_unfront (torch.profiler) in the put of a DELTA_BYTE_ARRAY part whose sorted
values share long prefixes ("/usr/lib/python3/site-packages/module_0000123/frame_4").

    python scripts/plain_strings_upload.py [--rows N] [--reps K] [--out FILE]
"""
import argparse
import io
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from frostdb_b200 import dynparquet as dp  # noqa: E402
from frostdb_b200 import logicalplan as lp  # noqa: E402
from frostdb_b200 import query  # noqa: E402
from frostdb_b200.store import ColumnStore  # noqa: E402

SCHEMA = dp.Schema(name="upload", columns=[dp.ColumnDefinition("s", dp.TYPE_STRING), dp.ColumnDefinition("timestamp", dp.TYPE_INT64),
                                           dp.ColumnDefinition("value", dp.TYPE_INT64)],
                   sorting_columns=[dp.SortingColumn("timestamp")])


def make_table(n_rows: int, n_distinct: int, seed: int) -> pa.Table:
    rng = np.random.default_rng(seed)
    ids = rng.permutation(n_rows) % n_distinct if n_distinct < n_rows else rng.permutation(n_rows)
    width = len(str(n_distinct))
    s = pa.array([f"stack/{i:0{width}d}/frame" for i in ids.tolist()], type=pa.string())
    t = pa.table({"s": s, "timestamp": pa.array(np.arange(n_rows, dtype=np.int64)),
                  "value": pa.array(rng.integers(0, 1000, n_rows))})
    return t.replace_schema_metadata({"dynamic_columns": ""})


def parquet(t: pa.Table, dictionary: bool, encoding: str = None) -> bytes:
    sink = io.BytesIO()
    kwargs = {"column_encoding": {"s": encoding}} if encoding else {}
    pq.write_table(t, sink, compression="NONE", use_dictionary=["s"] if dictionary else False, dictionary_pagesize_limit=1 << 30,
                   row_group_size=t.num_rows, store_schema=False, **kwargs)
    return sink.getvalue()


def unfront_time(cs, db, n_rows: int) -> dict:
    """k_str_unfront's device time in the put of a sorted DELTA_BYTE_ARRAY part with long shared prefixes."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    s = pa.array([f"/usr/lib/python3/site-packages/module_{i // 5:07d}/frame_{i % 5}" for i in range(n_rows)], type=pa.string())
    t = pa.table({"s": s, "timestamp": pa.array(np.arange(n_rows, dtype=np.int64)), "value": pa.array(np.zeros(n_rows, dtype=np.int64))})
    buf = parquet(t.replace_schema_metadata({"dynamic_columns": ""}), False, "DELTA_BYTE_ARRAY")
    torch.cuda.init()
    out = {}
    for rep in ("warm", "measured"):
        name = f"unfront_{rep}"
        db.Table(name, SCHEMA)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            cs.engine.put_parquet(name, buf)
        cs.engine.drop_table(name)
        db.tables.pop(name, None)
        us = {}
        for e in prof.events():
            if e.device_type.name == "CUDA" and "k_str_" in e.name:
                k = e.name.split("k_str_")[1].split("(")[0].split("E")[0]
                us["k_str_" + k] = us.get("k_str_" + k, 0.0) + e.device_time
        out = {"rows": n_rows, "rebuilt_bytes": sum(len(v) for v in s.to_pylist()),
               "kernel_us": {k: round(v, 1) for k, v in sorted(us.items())}}
    return out


def record(t: pa.Table) -> pa.RecordBatch:
    t = t.combine_chunks()
    return pa.RecordBatch.from_arrays([t.column(n).chunk(0).cast(pa.binary()) if n == "s" else t.column(n).chunk(0)
                                       for n in t.column_names], names=t.column_names)


def execute(db, table: str) -> int:
    out = []
    plan = query.NewEngine(None, db.TableProvider()).ScanTable(table).Filter(lp.Col("s").NotEq(lp.Literal("none")))
    plan.Aggregate([lp.Count(lp.Col("value"))], []).Execute(None, lambda c, r: out.append(r))
    return sum(b.column(0).to_pylist()[0] for b in out if b.num_rows)


def card() -> dict:
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        name, power = [x.strip() for x in q.stdout.strip().splitlines()[0].split(",")]
        return {"gpu": name, "power_limit": power}
    except Exception as e:  # (the numbers are still reported, without the card)
        return {"gpu": f"unknown ({e})", "power_limit": "unknown"}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=4 << 20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the result JSON to this file")
    args = ap.parse_args()
    cs = ColumnStore(0)
    db = cs.DB(None, "upload")
    results = []
    k = 0
    for n_distinct in (16, 64 << 10, args.rows):
        t = make_table(args.rows, n_distinct, 7)
        inputs = {"plain": parquet(t, False), "dlba": parquet(t, False, "DELTA_LENGTH_BYTE_ARRAY"),
                  "dba": parquet(t, False, "DELTA_BYTE_ARRAY"), "dictionary": parquet(t, True), "arrow": record(t)}
        for rep, src in inputs.items():
            k += 1
            name = f"u{k}"
            db.Table(name, SCHEMA)
            t0 = time.perf_counter()
            if rep == "arrow":
                cs.engine.put_arrow(name, src)
            else:
                cs.engine.put_parquet(name, src)
            t1 = time.perf_counter()
            n = execute(db, name)
            t2 = time.perf_counter()
            assert n == args.rows, (rep, n_distinct, n)
            steady = []
            for _ in range(args.reps):
                a = time.perf_counter()
                execute(db, name)
                steady.append(time.perf_counter() - a)
            assert cs.engine.dict_export(name, "s")[:3] == [v.encode() for v in dict.fromkeys(t.column("s")[:64].to_pylist())][:3]
            results.append({"distinct": n_distinct, "rep": rep, "put_ms": round((t1 - t0) * 1e3, 2),
                            "put_first_execute_ms": round((t2 - t0) * 1e3, 2), "steady_execute_ms": round(statistics.median(steady) * 1e3, 3)})
            print(json.dumps(results[-1]), flush=True)
            cs.engine.drop_table(name)
            db.tables.pop(name, None)
    try:
        unfront = unfront_time(cs, db, args.rows)
    except Exception as e:  # (the upload numbers are still reported)
        unfront = {"error": repr(e)}
    print(json.dumps({"unfront": unfront}), flush=True)
    cs.Close()
    out = {"rows": args.rows, **card(), "results": results, "unfront": unfront}
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
