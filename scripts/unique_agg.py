"""What a Unique(int64) aggregate costs in k_scan: bench_data-shaped parts plus an int64 column `u` that is constant per
labels.l00 value except for a seeded few rows, aggregated by two labels with the specialised kernels switched off
(FROSTGPU_NO_RUNS / NO_TILE / NO_PREFIX / NO_FAST), so that every plan runs in k_scan's general path.  Each plan is a
prepared query executed `--reps` times after one warm-up Execute (the cached path), reported as the median
scan_kernel_ms and total_device_ms:

  (a) Sum(value)                  the baseline
  (b) Sum(value), Unique(u)       two stored cells, almost every group has a value
  (c) Sum(value), Unique(value)   almost every group is NULL
  (d) Sum(value), Min(u), Max(u)  the Min / Max pair Unique is built from

    python scripts/unique_agg.py [--rows 32000000] [--reps 20] [--out DIR]

Prints one JSON object (and writes it to DIR/unique_agg.json when --out is given).  The part files go to a temporary
directory, never into the tree.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

for _switch in ("FROSTGPU_NO_RUNS", "FROSTGPU_NO_TILE", "FROSTGPU_NO_PREFIX", "FROSTGPU_NO_FAST"):
    os.environ[_switch] = "1"

import bench_data as bd  # noqa: E402
from frostdb_b200 import _lib  # noqa: E402
from frostdb_b200 import dynparquet as dp  # noqa: E402
from frostdb_b200 import logicalplan as lp  # noqa: E402
from frostdb_b200.physicalplan import GPUScan  # noqa: E402
from frostdb_b200.store import GPUEngine  # noqa: E402

N_LABELS = 4
PLANS = {
    "a: sum(value)": [lp.Sum(lp.Col("value"))],
    "b: sum(value), unique(u)": [lp.Sum(lp.Col("value")), lp.Unique(lp.Col("u"))],
    "c: sum(value), unique(value)": [lp.Sum(lp.Col("value")), lp.Unique(lp.Col("value"))],
    "d: sum(value), min(u), max(u)": [lp.Sum(lp.Col("value")), lp.Min(lp.Col("u")), lp.Max(lp.Col("u"))],
}


def part(first_row: int, n: int, cards) -> bytes:
    cols = bd.part_columns(first_row, n, N_LABELS, cards)
    l00 = cols["labels.l00"][0].astype(np.int64)
    i = np.arange(first_row, first_row + n, dtype=np.uint64)
    other = (bd.u(400, i) % np.uint64(1_000_000)) == 0  # about one row in a million differs from its l00 group
    cols["u"] = l00 * 1_000_003 + other.astype(np.int64)
    schema = dp.SampleDefinition()
    schema.columns.append(dp.ColumnDefinition("u", dp.TYPE_INT64))
    return dp.write_part(schema, cols, sort=False, row_group_size=bd.RG_ROWS)


def measure(eng, lib, aggs, reps):
    keys = [lp.Col("labels.l00"), lp.Col("labels.l01")]
    scan = GPUScan(eng, "t", None, _lib.PLAN_AGGREGATE, keys, aggs)
    q, keep = scan.prepare()
    kern, dev, st, nulls = [], [], None, 0
    try:
        for i in range(reps + 1):
            res = C.c_void_p()
            _lib.check(lib.fgpu_query_execute(eng.handle, q, eng.table_watermark("t"), C.byref(res)))
            try:
                recs = list(eng.drain(res))
                st = eng.stats(res)
            finally:
                lib.fgpu_result_free(res)
            if i:
                kern.append(st["scan_kernel_ms"])
                dev.append(st["total_device_ms"])
            nulls = sum(r.column(r.num_columns - 1).null_count for r in recs)
    finally:
        lib.fgpu_query_free(q)
        del keep
    n_rg = int(st["row_groups"]) - int(st["row_groups_pruned"])
    k_scan = n_rg - int(st["row_groups_runs"]) - int(st["row_groups_tiles"])
    return {"scan_kernel_ms": round(float(np.median(kern)), 4), "total_device_ms": round(float(np.median(dev)), 4),
            "groups": int(st["groups"]), "null_groups_last_column": int(nulls), "row_groups": n_rg, "k_scan_row_groups": k_scan}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=32_000_000)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    try:  # what the numbers were measured on
        gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True).stdout.strip()
    except OSError:
        gpu = "unknown"
    lib = _lib.load()
    cards = bd.cardinalities(N_LABELS)
    eng = GPUEngine(0)
    try:
        with tempfile.TemporaryDirectory() as d:
            for r in range(0, a.rows, bd.PART_ROWS):
                path = os.path.join(d, "part.parquet")
                with open(path, "wb") as f:
                    f.write(part(r, min(bd.PART_ROWS, a.rows - r), cards))
                eng.put_parquet("t", np.fromfile(path, dtype=np.uint8))
        out = {"gpu": gpu, "rows": a.rows, "reps": a.reps, "keys": "labels.l00, labels.l01",
               "plans": {name: measure(eng, lib, aggs, a.reps) for name, aggs in PLANS.items()}}
    finally:
        eng.close()
    text = json.dumps(out, indent=1)
    print(text)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "unique_agg.json"), "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
