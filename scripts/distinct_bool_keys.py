"""What a boolean Distinct key costs in k_scan: three Distinct shapes on bench_data's parts (100 M rows by default),
each a prepared query executed `--reps` times after one warm-up Execute (the cached path), reported as the median
scan_kernel_ms and total_device_ms with the kernels that took the row groups.

    python scripts/distinct_bool_keys.py [--rows 100000000] [--reps 20] [--out DIR]

Prints one JSON object (and writes it to DIR/distinct_bool_keys.json when --out is given).  The part files go to
bench_data's scratch directory (/dev/shm or /tmp), never into the tree.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench_data as bd  # noqa: E402
from frostdb_b200 import _lib  # noqa: E402
from frostdb_b200 import logicalplan as lp  # noqa: E402
from frostdb_b200.physicalplan import GPUScan  # noqa: E402
from frostdb_b200.store import GPUEngine  # noqa: E402

N_LABELS = 16


def shapes(rows: int):
    l00, l01 = lp.Col("labels.l00"), lp.Col("labels.l01")
    return {
        "distinct(l00, l01)": [l00, l01],
        "distinct(l00, l01, value > 500)": [l00, l01, lp.Col("value").Gt(lp.Literal(500))],
        # the statistics decide the key on every row group but the one holding the middle row
        "distinct(example_type, l00, timestamp > T0 + N/2)": [lp.Col("example_type"), l00,
                                                             lp.Col("timestamp").Gt(lp.Literal(bd.T0 + rows // 2))],
    }


def measure(eng, lib, table, keys, reps):
    scan = GPUScan(eng, table, None, _lib.PLAN_DISTINCT, keys, [])
    q, keep = scan.prepare()
    kern, dev, st = [], [], None
    try:
        for i in range(reps + 1):
            res = C.c_void_p()
            _lib.check(lib.fgpu_query_execute(eng.handle, q, eng.table_watermark(table), C.byref(res)))
            try:
                for _ in eng.drain(res):
                    pass
                st = eng.stats(res)
            finally:
                lib.fgpu_result_free(res)
            if i:
                kern.append(st["scan_kernel_ms"])
                dev.append(st["total_device_ms"])
    finally:
        lib.fgpu_query_free(q)
        del keep
    n_rg = int(st["row_groups"]) - int(st["row_groups_pruned"])
    runs, tiles = int(st["row_groups_runs"]), int(st["row_groups_tiles"])
    return {"scan_kernel_ms": round(float(np.median(kern)), 4), "total_device_ms": round(float(np.median(dev)), 4),
            "groups": int(st["groups"]), "row_groups": n_rg,
            "routing": {"k_runs_tma": runs - int(st["row_groups_prefix"]), "k_runs_prefix": int(st["row_groups_prefix"]),
                        "k_tile_agg": tiles, "k_scan": n_rg - runs - tiles}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    try:  # what the numbers were measured on
        gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True).stdout.strip()
    except OSError:
        gpu = "unknown"
    lib = _lib.load()
    eng = GPUEngine(0)
    try:
        for p in bd.generate_parts(a.rows, N_LABELS):
            eng.put_parquet("t", np.fromfile(p, dtype=np.uint8))
        out = {"gpu": gpu, "rows": a.rows, "reps": a.reps,
               "shapes": {name: measure(eng, lib, "t", keys, a.reps) for name, keys in shapes(a.rows).items()}}
    finally:
        eng.close()
    text = json.dumps(out, indent=1)
    print(text)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "distinct_bool_keys.json"), "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
