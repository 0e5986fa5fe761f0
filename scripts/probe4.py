"""Probe of the sorted-run kernels k_runs_tma / k_runs_prefix on PROBE_ROWS (default 32 Mi) sorted rows (runs on a GPU):
kernel time of a set of plan shapes with and without the prefix path (FROSTGPU_NO_PREFIX), then a sweep of tile bytes /
ring stages / consumer warps / chunk tiles (FROSTGPU_RT_*), every result compared row by row with the default shape's."""
import ctypes as C, os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import pyarrow as pa
import bench_data as bd
from frostdb_b200 import _lib, logicalplan as lp
from frostdb_b200.physicalplan import GPUScan
from frostdb_b200.store import GPUEngine

rows = int(os.environ.get("PROBE_ROWS", 32 * 1024 * 1024))
lib = _lib.load()
eng = GPUEngine(0)
ONLY = os.environ.get("PROBE_ONLY")


def load(table, sort):
    paths = bd.generate_parts(rows, 16, sort=sort)[: rows // bd.PART_ROWS]
    for p in paths:
        eng.put_parquet(table, np.fromfile(p, dtype=np.uint8))


def digest(batches):
    t = pa.Table.from_batches(batches)
    cols = []
    for name in t.column_names:
        c = t.column(name).combine_chunks()
        if pa.types.is_dictionary(c.type):
            c = c.cast(pa.string()) if not pa.types.is_binary(c.type.value_type) else c.dictionary_decode().cast(pa.binary())
        cols.append(c.to_pylist())
    return sorted(zip(*cols), key=lambda r: tuple((x is None, x) for x in r)) if cols else []


results = {}


def run(table, name, kind, f, groups, aggs, env=None):
    env = env or {}
    tag = " ".join(f"{a.replace('FROSTGPU_', '')}={b}" for a, b in env.items())
    if ONLY and ONLY not in name + " " + tag:
        return
    os.environ.update(env)
    try:
        scan = GPUScan(eng, table, f, kind, groups, aggs)
        q, keep = scan.prepare()
        ms, wall = [], []
        for i in range(int(os.environ.get("PROBE_REPS", 6))):
            res = C.c_void_p()
            t0 = time.perf_counter()
            _lib.check(lib.fgpu_query_execute(eng.handle, q, eng.table_watermark(table), C.byref(res)))
            wall.append((time.perf_counter() - t0) * 1e3)
            st = eng.stats(res)
            if i == 0:
                got = digest(list(eng.drain(res)))
            lib.fgpu_result_free(res)
            ms.append(st["scan_kernel_ms"])
        k = min(ms[1:])
        ref = results.setdefault((table, name), got)
        same = "same" if ref == got else "DIFFERENT"
        print(f"{name:44s} {tag:30s} kernel_ms {k:7.4f} exec_ms {min(wall[1:]):7.3f} GB/s {st['algorithmic_bytes'] / k / 1e6:7.1f} "
              f"sel {st['rows_selected']:>9d} groups {st['groups']:>6d} rg prefix/runs/tiles/all {st['row_groups_prefix']}/{st['row_groups_runs']}/{st['row_groups_tiles']}/{st['row_groups']} {same}", flush=True)
        lib.fgpu_query_free(q)
    finally:
        for a in env:
            os.environ.pop(a)


ts, val, fval = lp.Col("timestamp"), lp.Col("value"), lp.Col("floatvalue")
K01 = [lp.Col("labels.l00"), lp.Col("labels.l01")]
AGG = _lib.PLAN_AGGREGATE
load("s", True)
F50 = lp.And(ts.GtEq(lp.Literal(bd.T0 + rows // 4)), ts.Lt(lp.Literal(bd.T0 + 3 * rows // 4)))
VF = val.Lt(lp.Literal(500))
cases = [
    ("sorted: sum by l00,l01", None, K01, [lp.Sum(val)]),
    ("sorted: ts 50%, sum,count by l00,l01", F50, K01, [lp.Sum(val), lp.Count(val)]),
    ("sorted: value<500, sum by l00,l01", VF, K01, [lp.Sum(val)]),
    ("sorted: value<500 & ts 50%, sum by l00,l01", lp.And(VF, F50), K01, [lp.Sum(val)]),
    ("sorted: sum (no keys)", None, [], [lp.Sum(val)]),
    ("sorted: value<500, sum (no keys)", VF, [], [lp.Sum(val)]),
    ("sorted: sum by l00", None, K01[:1], [lp.Sum(val)]),
    ("sorted: count by l00,l01", None, K01, [lp.Count(val)]),
    ("sorted: sum,min,max by l00,l01", None, K01, [lp.Sum(val), lp.Min(val), lp.Max(val)]),
    ("sorted: l00 == v000003, sum by l00,l01", lp.Col("labels.l00").Eq(lp.Literal("v000003")), K01, [lp.Sum(val)]),
    ("sorted: l01 != v000003, sum by l00,l01", lp.Col("labels.l01").NotEq(lp.Literal("v000003")), K01, [lp.Sum(val)]),
]
for name, f, g, a in cases:
    run("s", name, AGG, f, g, a)
    run("s", name, AGG, f, g, a, {"FROSTGPU_NO_PREFIX": "1"})  # the same row groups through k_runs_tma
if os.environ.get("PROBE_NOSWEEP"):
    sys.exit(0)
def sweep(ci, combos):
    for t, st, w, sp in combos:
        env = {}
        if t: env["FROSTGPU_RT_TILE"] = str(t)  # tile bytes / 8
        if st: env["FROSTGPU_RT_STAGES"] = str(st)
        if w: env["FROSTGPU_RT_WARPS"] = str(w)
        if sp: env["FROSTGPU_RT_SPAN"] = str(sp)
        run("s", cases[ci][0], AGG, cases[ci][1], cases[ci][2], cases[ci][3], env)


for ci in (1, 0, 2):
    sweep(ci, [(t, st, 0, sp) for t in (2048, 4096, 8192) for st in (2, 3, 4) for sp in (1, 2, 4, 8)] + [(4096, 2, 4, 4), (2048, 3, 4, 2)])
