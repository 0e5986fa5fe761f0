"""Device time of the general kernels that decode hybrid column chunks outside k_scan (runs on a GPU).

  python scripts/general_decode.py [--rows 16777216] [--reps 20] [--out DIR]

bench_data parts in arrival order (unsorted, 4 labels: l00 / l01 without NULLs, l02 / l03 with about 10 % NULLs):

  k_rows     a filter-only plan under FROSTGPU_NO_TAKE=1 that projects labels.l02 and value under an OR filter
             (value < 100 OR labels.l01 == "v000007"); one prepared query executed --reps times
  k_decode   fgpu_part_decode_column of labels.l02 and of value on every part, --reps rounds
  k_flatten  the first Execute of Sum(value) GROUP BY labels.l00, labels.l01 (a tile plan, which flattens both key
             columns), on a fresh engine each of --reps rounds

Each kernel is timed by name with torch.profiler (CUDA activities) in a run of its own, after one untimed warm-up
round, and reported as the median of its per-round device time.  A sha256 digest of each case's outputs (the k_rows
record, the decoded arrays, the sorted aggregate rows) lets two builds be compared.  The card's name and power limit
are read in the same run.  Prints one JSON object (and writes it to DIR/general_decode.json when --out is given); the
part files go to bench_data's scratch directory, never into the tree.
"""
from __future__ import annotations

import argparse
import ctypes as C
import hashlib
import json
import os
import subprocess
import sys
from collections import defaultdict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import pyarrow as pa  # noqa: E402
import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

import bench_data as bd  # noqa: E402
from frostdb_b200 import _lib  # noqa: E402
from frostdb_b200 import logicalplan as lp  # noqa: E402
from frostdb_b200.physicalplan import GPUScan  # noqa: E402
from frostdb_b200.store import GPUEngine  # noqa: E402

N_LABELS = 4
KERNELS = ("k_rows", "k_decode", "k_flatten")


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def kernel_ms(prof):
    """{kernel: total device ms} of the named kernels in one profile."""
    tot = defaultdict(float)
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA and e.device_time > 0:
            name = e.name.replace("fgpu::", "").removeprefix("void ").split("(")[0].split("<")[0].strip()
            if name in KERNELS:
                tot[name] += e.device_time / 1e3
    return tot


def timed(fn, reps):
    """fn() once untimed, then reps rounds, each profiled on its own: ({kernel: median ms per round}, last output)."""
    out = fn()
    torch.cuda.synchronize()
    per = defaultdict(list)
    for _ in range(reps):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            out = fn()
            torch.cuda.synchronize()
        for k, v in kernel_ms(prof).items():
            per[k].append(v)
    return {k: round(float(np.median(v)), 4) for k, v in sorted(per.items())}, out


def digest_array(h, a):
    if isinstance(a, pa.ChunkedArray):
        a = a.combine_chunks()
    h.update(str(a.type).encode())
    if pa.types.is_dictionary(a.type):
        h.update(a.indices.cast(pa.int64()).fill_null(-1).to_numpy(zero_copy_only=False).tobytes())
        h.update("\0".join(str(v) for v in a.dictionary.to_pylist()).encode())
    else:
        h.update(a.is_null().to_numpy(zero_copy_only=False).tobytes())
        h.update(a.fill_null(0).to_numpy(zero_copy_only=False).tobytes())


def execute(eng, q, table):
    lib = _lib.load()
    res = C.c_void_p()
    _lib.check(lib.fgpu_query_execute(eng.handle, q, eng.table_watermark(table), C.byref(res)))
    try:
        return list(eng.drain(res)), eng.stats(res)
    finally:
        lib.fgpu_result_free(res)


def load(paths):
    eng = GPUEngine(0)
    for p in paths:
        eng.put_parquet("t", np.fromfile(p, dtype=np.uint8))
    return eng


def case_rows(paths, reps):
    os.environ["FROSTGPU_NO_TAKE"] = "1"
    eng = load(paths)
    try:
        names = ["labels.l02", "value"]
        filt = lp.Or(lp.Col("value").Lt(lp.Literal(100)), lp.Col("labels.l01").Eq(lp.Literal("v000007")))
        q, keep = GPUScan(eng, "t", filt, _lib.PLAN_FILTER, [lp.Col(n) for n in names], []).prepare()
        try:
            ms, (batches, st) = timed(lambda: execute(eng, q, "t"), reps)
        finally:
            _lib.load().fgpu_query_free(q)
            del keep
        h = hashlib.sha256()
        for b in batches:
            for col in b.columns:
                digest_array(h, col)
        return {"ms": ms, "rows_selected": int(st["rows_selected"]), "digest": h.hexdigest()[:16]}
    finally:
        eng.close()
        os.environ.pop("FROSTGPU_NO_TAKE")


def case_decode(paths, reps):
    eng = load(paths)
    try:
        def run():
            return [eng.decode_column("t", pid, col) for pid in range(len(paths)) for col in ("labels.l02", "value")]
        ms, arrays = timed(run, reps)
        h = hashlib.sha256()
        for a in arrays:
            digest_array(h, a)
        return {"ms": ms, "digest": h.hexdigest()[:16]}
    finally:
        eng.close()


def case_flatten(paths, reps):
    def run():  # a fresh engine: its first tile-plan Execute builds the flat code images
        eng = load(paths)
        try:
            q, keep = GPUScan(eng, "t", None, _lib.PLAN_AGGREGATE, [lp.Col("labels.l00"), lp.Col("labels.l01")],
                              [lp.Sum(lp.Col("value"))]).prepare()
            try:
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    batches, st = execute(eng, q, "t")
                    torch.cuda.synchronize()
            finally:
                _lib.load().fgpu_query_free(q)
                del keep
        finally:
            eng.close()
        rows = sorted((tuple(r.values()) for b in batches for r in b.to_pylist()), key=repr)
        return kernel_ms(prof), rows, int(st["row_groups_tiles"])

    run()
    per = defaultdict(list)
    for _ in range(reps):
        ms, rows, tiles = run()
        for k, v in ms.items():
            per[k].append(v)
    h = hashlib.sha256(repr(rows).encode())
    return {"ms": {k: round(float(np.median(v)), 4) for k, v in sorted(per.items())}, "row_groups_tiles": tiles,
            "groups": len(rows), "digest": h.hexdigest()[:16]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=4 * bd.PART_ROWS)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    torch.cuda.set_device(0)
    paths = bd.generate_parts(a.rows, N_LABELS, sort=False)
    out = {"card": card(), "rows": a.rows, "reps": a.reps,
           "k_rows": case_rows(paths, a.reps), "k_decode": case_decode(paths, a.reps),
           "k_flatten": case_flatten(paths, a.reps)}
    text = json.dumps(out)
    print(text)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "general_decode.json"), "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
