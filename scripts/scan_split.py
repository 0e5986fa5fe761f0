"""Per-launch time of a cached aggregate Execute on SPLIT_ROWS (default 100 M) sorted rows (runs on a GPU).

  python scripts/scan_split.py [OUT_DIR]

Three prepared queries on the bench.py table: the headline (timestamp in the middle 50 %, Sum(value), Count(value) GROUP
BY l00, l01), cfg3_sorted_nofilter (the same without filter) and `sum by l01` (a key that is not a sort prefix).  Each is
executed a few times to warm up, then SPLIT_REPS times under torch.profiler with CUDA activities; the line of a query
gives every kernel's mean device time per Execute, and the first (uncached) Execute's kernels on their own.  The card's
name and power limit go into the JSON written to OUT_DIR/scan_split.json."""
import ctypes as C
import json
import os
import subprocess
import sys
import time
from collections import defaultdict

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from torch.profiler import ProfilerActivity, profile

import bench_data as bd
from frostdb_b200 import _lib, logicalplan as lp
from frostdb_b200.physicalplan import GPUScan
from frostdb_b200.store import GPUEngine

rows = int(os.environ.get("SPLIT_ROWS", 100_000_000))
reps = int(os.environ.get("SPLIT_REPS", 200))
out_dir = sys.argv[1] if len(sys.argv) > 1 else None


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def kernel_times(prof, n):
    """{kernel name: mean ms per Execute} over the device kernels of a profile of n Executes."""
    tot = defaultdict(float)
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA and e.device_time > 0:
            name = e.name.replace("(anonymous namespace)::", "").replace("fgpu::", "").removeprefix("void ")
            tot[name.split("(")[0].split("<")[0].strip() or e.name] += e.device_time
    return {k: round(v / 1e3 / n, 5) for k, v in sorted(tot.items(), key=lambda kv: -kv[1])}


def execute(eng, lib, q, tx):
    res = C.c_void_p()
    _lib.check(lib.fgpu_query_execute(eng.handle, q, tx, C.byref(res)))
    st = eng.stats(res)
    lib.fgpu_result_free(res)
    return st


def main():
    torch.cuda.set_device(0)
    lib = _lib.load()
    eng = GPUEngine(0)
    for p in bd.generate_parts(rows, 16):
        eng.put_parquet("bench", np.fromfile(p, dtype=np.uint8))
    tx = eng.table_watermark("bench")
    ts, val = lp.Col("timestamp"), lp.Col("value")
    K01 = [lp.Col("labels.l00"), lp.Col("labels.l01")]
    f50 = lp.And(ts.GtEq(lp.Literal(bd.T0 + rows // 4)), ts.Lt(lp.Literal(bd.T0 + (3 * rows) // 4)))
    cases = [("headline", f50, K01, [lp.Sum(val), lp.Count(val)]),
             ("cfg3_sorted_nofilter", None, K01, [lp.Sum(val), lp.Count(val)]),
             ("sum_by_l01", None, [lp.Col("labels.l01")], [lp.Sum(val)])]
    out = {"card": card(), "rows": rows, "reps": reps, "cases": {}}
    for name, f, g, a in cases:
        q, keep = GPUScan(eng, "bench", f, _lib.PLAN_AGGREGATE, g, a).prepare()
        with profile(activities=[ProfilerActivity.CUDA]) as p0:
            st0 = execute(eng, lib, q, tx)  # the first Execute compiles the plan
            torch.cuda.synchronize()
        for _ in range(5):
            execute(eng, lib, q, tx)
        torch.cuda.synchronize()
        wall = []
        scan = []
        for _ in range(reps):
            t0 = time.perf_counter()
            st = execute(eng, lib, q, tx)
            wall.append((time.perf_counter() - t0) * 1e3)
            scan.append(st["scan_kernel_ms"])
        with profile(activities=[ProfilerActivity.CUDA]) as p:
            for _ in range(reps):
                execute(eng, lib, q, tx)
            torch.cuda.synchronize()
        line = {"kernels_per_execute_ms": kernel_times(p, reps), "first_execute_kernels_ms": kernel_times(p0, 1),
                "scan_kernel_ms_median": round(float(np.median(scan)), 5), "exec_ms_median": round(float(np.median(wall)), 5),
                "kernel_launches": int(st["kernel_launches"]), "row_groups_prefix": int(st["row_groups_prefix"]),
                "row_groups_runs": int(st["row_groups_runs"]), "row_groups_tiles": int(st["row_groups_tiles"]),
                "algorithmic_bytes": int(st["algorithmic_bytes"]), "rows_selected": int(st["rows_selected"]),
                "first_exec_rows_selected": int(st0["rows_selected"])}
        out["cases"][name] = line
        print(name, json.dumps(line), flush=True)
        lib.fgpu_query_free(q)
    print("card", out["card"], flush=True)
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        with open(os.path.join(out_dir, "scan_split.json"), "w") as fh:
            json.dump(out, fh, indent=1)
    eng.close()


if __name__ == "__main__":
    main()
