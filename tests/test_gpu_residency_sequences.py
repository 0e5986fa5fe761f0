"""Lazily built column images in every order that puts, queries, decodes, refusals and drops can build them
(tests/residency_model.py holds the parts, the plans, the reference and the sequence generator).  After every query:

1. the records equal the reference;
2. they equal the cold answer: a fresh table of the same store with the same visible parts put eagerly (Arrow parts as
   Arrow), compared by key (group order follows dictionary ids), values bit for bit, and so do the routing stats;
3. every string column's dict_export lists each string once, extends the previous step's list (an id never changes
   meaning) and holds the strings of every column made resident whole (eager puts, decodes, unfiltered keys);
4. running the same prepared query again at once gives the same records and copies only its plan's descriptors: what
   a third run copies, where every column the plan reads is resident, and nothing for a cached dense plan;
5. every result record still held gives the values it gave when it was returned, after every later query;
6. a refused query fails with the same code and message each time, and everything after the corrupted part's drop
   matches the reference.

RESIDENCY_WALK_SEEDS / RESIDENCY_WALK_STEPS widen the seeded walks."""
import ctypes as C
import os
import re
import struct

import numpy as np
import pyarrow as pa
import pytest

from frostdb_b200 import _lib
from frostdb_b200 import logicalplan as lp
from frostdb_b200.physicalplan import GPUScan
from tests import delta_int64 as di
from tests import delta_strings as ds
from tests import numeric_edges as ne
from tests import residency_model as m

pytestmark = pytest.mark.gpu

ROUTE = ("row_groups_runs", "row_groups_prefix", "row_groups_tiles", "row_groups", "row_groups_pruned", "rows_selected")
DICT_COLUMNS = m.STRINGS + [m.LABEL]
KIND = {"agg": _lib.PLAN_AGGREGATE, "distinct": _lib.PLAN_DISTINCT, "rows": _lib.PLAN_FILTER}
BANK = m.bank()
PLAN = {p.name: i for i, p in enumerate(BANK)}
SEEDS = int(os.environ.get("RESIDENCY_WALK_SEEDS", "16"))
STEPS = int(os.environ.get("RESIDENCY_WALK_STEPS", "30"))


@pytest.fixture(autouse=True)
def clean_switches():
    yield
    for k in m.SWITCHES:
        os.environ.pop(k, None)


def _strings(a) -> list:
    if isinstance(a, pa.ChunkedArray):
        a = pa.concat_arrays(a.chunks) if a.num_chunks else pa.array([], a.type)
    if pa.types.is_dictionary(a.type):
        a = a.dictionary_decode()
    return [x.decode() if isinstance(x, bytes) else x for x in a.to_pylist()]


def _canon(x):
    """Floats by their bits: -0.0 and +0.0 differ."""
    if isinstance(x, float):
        return ("f", struct.unpack("<q", struct.pack("<d", x))[0])
    if isinstance(x, tuple):
        return tuple(_canon(v) for v in x)
    return x


def parse(plan: m.Plan, batches):
    """Aggregates as {key: values}, Distinct as a set of tuples (the all-NULL tuple aside), rows as a list."""
    batches = [b for b in batches if b.num_rows]
    if plan.kind == "agg":
        return {_canon(k): _canon(v) for k, v in ne.result_map(batches, plan.keys, plan.aggs).items()}
    rows = []
    for b in batches:  # (a record of parts that lack a projected column has no such column: NULL)
        cols = [b.schema.get_field_index(n) for n in plan.keys]
        rows.extend(zip(*[_strings(b.column(i)) if i >= 0 else [None] * b.num_rows for i in cols]))
    if plan.kind == "distinct":
        return {r for r in rows if r != (None,) * len(plan.keys)}
    return [_canon(r) for r in rows]


def assert_reference(plan: m.Plan, got, exp, what: str, float_groups=frozenset()):
    if plan.kind == "distinct":
        assert got == exp, f"{what}: distinct differs: {sorted(got ^ exp, key=str)[:5]}"
        return
    if plan.kind == "rows":
        exp = [_canon(r) for r in exp]
        assert len(got) == len(exp), f"{what}: {len(got)} rows, expected {len(exp)}"
        bad = next((i for i, (g, e) in enumerate(zip(got, exp)) if g != e), None)
        assert bad is None, f"{what}: row {bad}: got {got[bad]!r}, expected {exp[bad]!r}"
        return
    exp = {_canon(k): v for k, v in exp.items()}
    assert set(got) == set(exp), f"{what}: groups differ: {sorted(set(got) ^ set(exp), key=str)[:5]}"
    for k, ev in exp.items():
        for a, g, e in zip(plan.aggs, got[k], ev):
            if isinstance(e, float) and a.Func == lp.AggFuncSum and g is None and k not in float_groups:
                continue  # a group whose floatvalue is NULL throughout (Sum of no value: NULL or 0.0)
            assert _canon(e) == g, f"{what}: group {k} {a.Name()}: got {g!r}, expected {e!r}"


class Walk:
    """One table of the store driven through a sequence of operations, checked after each one."""

    def __init__(self, store, table: str, what: str):
        self.store, self.eng, self.lib = store, store.engine, _lib.load()
        self.table, self.what = table, what
        self.visible = []  # (part id, part name, how) in put order
        self.keep = []     # borrowed buffers (kept until the store goes)
        self.prepared = {}
        self.held = []     # (what, records, parsed) of every query run
        self.dicts = {c: [] for c in DICT_COLUMNS}
        self.must = {c: set() for c in DICT_COLUMNS}
        self.cold = {}
        self.n_cold = 0
        self._drop_table(table)

    def _drop_table(self, table):
        try:
            self.eng.drop_table(table)
        except _lib.FrostGPUError:
            pass

    def close(self):
        for q, _ in self.prepared.values():
            self.lib.fgpu_query_free(q)
        self.prepared.clear()
        self._drop_table(self.table)

    # ---- execution ----
    def _prepare(self, table, plan):
        return GPUScan(self.eng, table, plan.filt, KIND[plan.kind], [lp.Col(k) for k in plan.keys], list(plan.aggs)).prepare()

    def _execute(self, table, q):
        res = C.c_void_p()
        _lib.check(self.lib.fgpu_query_execute(self.eng.handle, q, self.eng.table_watermark(table), C.byref(res)))
        try:
            batches = list(self.eng.drain(res))
            st = self.eng.stats(res)
        finally:
            self.lib.fgpu_result_free(res)
        return batches, st

    def _cold(self, i, plan):
        key = (tuple((name, how == "arrow") for _, name, how in self.visible), i, tuple(os.environ.get(k) for k in m.SWITCHES))
        if key not in self.cold:
            table = f"{self.table}_cold{self.n_cold}"
            self.n_cold += 1
            self._drop_table(table)
            try:
                for _, name, how in self.visible:
                    if how == "arrow":
                        self.eng.put_arrow(table, m.record_of(name))
                    else:
                        self.eng.put_parquet(table, m.file_of(name))
                q, _ = self._prepare(table, plan)
                try:
                    batches, st = self._execute(table, q)
                finally:
                    self.lib.fgpu_query_free(q)
                self.cold[key] = (parse(plan, batches), {k: st[k] for k in ROUTE})
            finally:
                self._drop_table(table)
        return self.cold[key]

    # ---- operations ----
    def put(self, name, how):
        if how == "arrow":
            pid = self.eng.put_arrow(self.table, m.record_of(name))
        else:
            arr = np.frombuffer(m.file_of(name), dtype=np.uint8)
            self.keep.append(arr)
            pid = self.eng.put_parquet(self.table, arr, borrow=how == "borrow")
        self.visible.append((pid, name, how))
        if how != "borrow":  # an eager or Arrow part interns every string column at its put
            for c in DICT_COLUMNS:
                if c in m.table_of(name).column_names:
                    self.must[c] |= {v for v in m.table_of(name).column(c).to_pylist() if v is not None}

    def drop(self, name):
        pid = next(p for p, n, _ in self.visible if n == name)
        self.eng.drop_part(self.table, pid)
        self.visible = [v for v in self.visible if v[0] != pid]

    def decode(self, name, column, what):
        pid = next(p for p, n, _ in self.visible if n == name)
        got = self.eng.decode_column(self.table, pid, column)
        exp = m.table_of(name).column(column).to_pylist()
        assert (_strings(got) if column in DICT_COLUMNS else got.to_pylist()) == exp, f"{what}: decode_column {name}.{column}"
        if column in DICT_COLUMNS:
            self.must[column] |= {v for v in exp if v is not None}

    def query(self, i, mode, what):
        plan = BANK[i]
        if mode == "fresh" or i not in self.prepared:
            if i in self.prepared:
                self.lib.fgpu_query_free(self.prepared.pop(i)[0])
            self.prepared[i] = self._prepare(self.table, plan)
        q = self.prepared[i][0]
        what = f"{what} plan {plan.name}"
        batches, st = self._execute(self.table, q)
        got = parse(plan, batches)
        self.held.append((what, batches, got))
        names = [n for _, n, _ in self.visible]
        floats = {_canon(k) for k in m.float_groups(plan, names)} if plan.kind == "agg" else set()
        assert_reference(plan, got, m.reference(plan, names), what + " vs reference", floats)
        cold, route = self._cold(i, plan)
        assert got == cold, f"{what}: differs from the cold answer"
        assert {k: st[k] for k in ROUTE} == route, f"{what}: routing {st} vs cold {route}"
        again, st2 = self._execute(self.table, q)
        self.held.append((what + " (again)", again, parse(plan, again)))
        assert self.held[-1][2] == got, f"{what}: the prepared query's second run differs"
        radix = 1
        for c in plan.keys:
            radix *= len(self._dict(c)) + 1 if c in DICT_COLUMNS else 1 << 32
        third = self._execute(self.table, q)[1]["h2d_bytes"]
        assert st2["h2d_bytes"] == third, f"{what}: the second run copied {st2['h2d_bytes']} bytes, the third {third}"
        if plan.cached and radix <= 65536:  # (a larger dense table is not kept between Executes)
            assert st2["h2d_bytes"] == 0, f"{what}: the cached second run copied {st2['h2d_bytes']} bytes"
        if plan.filt is None and plan.kind != "rows":  # every key column of every visible part is resident whole now
            for _, name, _ in self.visible:
                for c in plan.keys:
                    if c in DICT_COLUMNS and c in m.table_of(name).column_names:
                        self.must[c] |= {v for v in m.table_of(name).column(c).to_pylist() if v is not None}

    def corrupt(self, case, what):
        """A part whose `value` chunk breaks one DELTA_BINARY_PACKED rule (tests/delta_int64.py): a query reading it is
        refused the same way twice, then the part is dropped."""
        _, buf, message = next(c for c in di.corrupted() if c[0] == case)
        arr = np.frombuffer(buf, dtype=np.uint8)
        self.keep.append(arr)
        pid = self.eng.put_parquet(self.table, arr, borrow=True)
        plan = m.Plan("sum", "agg", (), (lp.Sum(m.V), lp.Count(m.V)))
        q, _ = self._prepare(self.table, plan)
        errors = []
        try:
            for _ in range(2):
                with pytest.raises(_lib.FrostGPUError) as e:
                    self._execute(self.table, q)
                errors.append((e.value.code, e.value.msg))
        finally:
            self.lib.fgpu_query_free(q)
        assert errors[0] == errors[1], f"{what}: {errors}"
        assert errors[0][0] == _lib.FGPU_ERR_UNSUPPORTED and "column value: " + message in errors[0][1], f"{what}: {errors[0]}"
        self.eng.drop_part(self.table, pid)

    def _dict(self, c):
        try:
            return [v.decode() for v in self.eng.dict_export(self.table, c)]
        except _lib.FrostGPUError:  # (no part of the table has interned the column yet)
            return []

    def check_dicts(self, what):
        for c in DICT_COLUMNS:
            d = self._dict(c)
            assert len(set(d)) == len(d), f"{what}: {c}: a string listed twice"
            prev = self.dicts[c]
            assert d[:len(prev)] == prev, f"{what}: {c}: the dictionary is not an extension of the previous step's"
            missing = self.must[c] - set(d)
            assert not missing, f"{what}: {c}: resident strings missing from the dictionary: {sorted(missing)[:3]}"
            self.dicts[c] = d

    def run(self, ops):
        for step, op in enumerate(ops):
            what = f"{self.what} step {step} {op}"
            kind = op[0]
            if kind == "put":
                self.put(op[1], op[2])
            elif kind == "drop":
                self.drop(op[1])
            elif kind == "decode":
                self.decode(op[1], op[2], what)
            elif kind == "query":
                self.query(op[1] if isinstance(op[1], int) else PLAN[op[1]], op[2], what)
            elif kind == "corrupt":
                self.corrupt(op[1], what)
            elif kind == "switch":
                if op[2]:
                    os.environ[op[1]] = "1"
                else:
                    os.environ.pop(op[1], None)
            self.check_dicts(what)
            if kind == "query":
                self.check_held(what)
        self.check_held(f"{self.what} end")

    def check_held(self, now):
        for what, batches, parsed in self.held:
            plan_name = re.search(r"plan (\w+)", what).group(1)
            assert parse(BANK[PLAN[plan_name]], batches) == parsed, f"{now}: a held result changed: {what}"

    def stats(self, plan):
        q, _ = self._prepare(self.table, plan)
        try:
            return self._execute(self.table, q)[1]
        finally:
            self.lib.fgpu_query_free(q)


def walk(store, table, what, ops):
    w = Walk(store, table, what)
    try:
        w.run(ops)
    finally:
        w.close()


# ---- hand-written orderings --------------------------------------------------------------------------------------
ORDERINGS = {
    "prune_then_full": [("put", "sorted_a", "borrow"), ("put", "unsorted_a", "borrow"), ("put", "edge", "borrow"),
                        ("query", "pruned", "fresh"), ("query", "hash_strings", "fresh"), ("query", "take", "fresh")],
    "decode_before_first_query": [("put", "sorted_c", "borrow"), ("decode", "sorted_c", "s_dba"), ("decode", "sorted_c", "value"),
                                  ("decode", "sorted_c", "s_plain"), ("query", "tile", "fresh"), ("query", "rows", "fresh"),
                                  ("query", "prefix", "fresh")],
    "refused_then_read": [("put", "sorted_a", "borrow"), ("put", "edge", "borrow"), ("corrupt", "bit_width"),
                          ("query", "hash_strings", "fresh"), ("corrupt", "count"), ("query", "scan_fast", "fresh"),
                          ("query", "distinct_pair", "fresh")],
    "prepared_after_dictionary_growth": [("put", "sorted_a", "borrow"), ("query", "tile", "fresh"), ("put", "edge", "borrow"),
                                         ("query", "tile", "prepared"), ("put", "unsorted_a", "arrow"), ("query", "tile", "prepared"),
                                         ("query", "rows", "fresh"), ("put", "short_runs", "borrow"), ("query", "rows", "prepared")],
    "drop_and_put_again": [("put", "sorted_b", "borrow"), ("put", "sorted_a", "eager"), ("query", "prefix", "fresh"),
                           ("drop", "sorted_b"), ("put", "sorted_b", "borrow"), ("query", "prefix", "prepared"),
                           ("query", "runs", "fresh"), ("drop", "sorted_a"), ("put", "sorted_a", "borrow"), ("query", "runs", "prepared")],
    "image_built_by_one_kernel_read_by_another": [
        ("put", "sorted_a", "borrow"), ("put", "sorted_c", "borrow"), ("query", "runs", "fresh"),
        ("switch", "FROSTGPU_NO_RUNS", True), ("query", "runs", "prepared"), ("query", "take_dict", "fresh"),
        ("switch", "FROSTGPU_NO_PREFIX", True), ("switch", "FROSTGPU_NO_RUNS", False), ("query", "prefix", "fresh"),
        ("switch", "FROSTGPU_NO_PREFIX", False), ("query", "prefix", "prepared"), ("query", "take", "fresh")],
    "arrow_and_borrowed_interleaved": [("put", "unsorted_a", "arrow"), ("put", "sorted_a", "borrow"), ("query", "distinct_pair", "fresh"),
                                       ("put", "edge", "arrow"), ("put", "sorted_c", "borrow"), ("query", "hash_strings", "fresh"),
                                       ("query", "rows", "fresh"), ("query", "scan_hash", "fresh"), ("query", "distinct", "fresh")],
    "edge_row_groups_and_widths": [("put", "edge", "borrow"), ("query", "tile", "fresh"), ("query", "rows", "fresh"),
                                   ("query", "distinct", "fresh"), ("decode", "edge", "s_plain"), ("decode", "edge", "s_dba"),
                                   ("put", "short_runs", "borrow"), ("query", "scan_fast", "fresh"), ("query", "take_dict", "fresh")],
    "flat_codes_of_three_widths_in_one_launch": [("put", "wide", "borrow"), ("query", "prefix", "fresh"), ("query", "take_dict", "fresh"),
                                                 ("put", "sorted_a", "borrow"), ("query", "prefix", "prepared"),
                                                 ("query", "tile_dict_leaf", "fresh"), ("query", "distinct_pair", "fresh"),
                                                 ("decode", "wide", "s_plain")],
}


@pytest.mark.parametrize("name", list(ORDERINGS))
def test_hand_written_ordering(store, name):
    walk(store, f"seq_{name}", name, ORDERINGS[name])


@pytest.mark.parametrize("seed", range(SEEDS))
def test_seeded_walk(store, seed):
    walk(store, f"walk_{seed}", f"seed {seed}", m.sequence(seed, STEPS))


def test_plans_take_the_kernels_they_aim_at(store):
    """On the sorted parts put eagerly: the run and prefix plans on the sorted-run kernels, the tile plan on the tile
    kernel, the pruned plan dropping the later parts whole; with the same plans on the unsorted part, no run kernel."""
    w = Walk(store, "seq_routes", "routes")
    try:
        for name in ("sorted_a", "sorted_c"):
            w.put(name, "eager")
        route = lambda p: w.stats(BANK[PLAN[p]])
        n_rg = sum(len(m.SPEC_BY_NAME[n].rgs) for n in ("sorted_a", "sorted_c"))
        st = route("prefix")
        assert st["row_groups_prefix"] == n_rg == st["row_groups_runs"], st
        st = route("runs")
        assert st["row_groups_runs"] == n_rg and st["row_groups_prefix"] < n_rg, st
        st = route("tile")
        assert st["row_groups_tiles"] == n_rg, st
        st = route("pruned")
        assert st["row_groups_pruned"] == len(m.SPEC_BY_NAME["sorted_c"].rgs), st
        w.put("unsorted_a", "eager")
        st = route("prefix")
        assert st["row_groups_runs"] == n_rg and st["row_groups_tiles"] == len(m.SPEC_BY_NAME["unsorted_a"].rgs), st
    finally:
        w.close()


def test_flat_codes_of_three_widths_go_to_one_tile_and_one_take_launch(store):
    """The wide part put first: its s_dict row groups hold global ids below 256, above 65 535 and in between, so their
    flat codes are 8, 32 and 16 bits wide.  A key on s_dict and a leaf on it take all three row groups to k_tile_agg;
    the filter-only plan with the leaf takes the ordered take kernels (two launches more than k_rows)."""
    w = Walk(store, "seq_wide_routes", "wide routes")
    try:
        w.put("wide", "eager")
        d = w._dict("s_dict")
        ids = {v: i for i, v in enumerate(d)}
        col = m.table_of("wide").column("s_dict").to_pylist()
        top = [max(ids[v] for v in col[lo:hi]) for lo, hi in m.row_group_bounds("wide")]
        assert top[0] < 256 and top[1] >= 65536 and 256 <= top[2] < 65536, top
        for name in ("prefix", "tile_dict_leaf"):
            st = w.stats(BANK[PLAN[name]])
            assert st["row_groups_tiles"] == len(m.WIDE_RGS) and st["row_groups_runs"] == 0, (name, st)
            w.query(PLAN[name], "fresh", f"wide routes plan {name}")
        take = w.stats(BANK[PLAN["take_dict"]])["kernel_launches"]
        os.environ["FROSTGPU_NO_TAKE"] = "1"
        try:
            rows = w.stats(BANK[PLAN["take_dict"]])["kernel_launches"]
        finally:
            os.environ.pop("FROSTGPU_NO_TAKE")
        assert take == rows + 2, (take, rows)
        w.query(PLAN["take_dict"], "fresh", "wide routes plan take_dict")
        w.check_held("wide routes end")
    finally:
        w.close()


def test_a_refused_query_leaves_its_walked_strings_to_the_next_querys_first_intern_batch(store):
    """upload_columns interns the listed columns already walked but not built before it walks the others (DESIGN.md
    §3).  A query refused on a corrupted DELTA_LENGTH_BYTE_ARRAY chunk (tests/delta_strings.py) leaves part X's `s`
    walked; the next query lists part Y (which the refused query pruned) first, yet X's strings take the first ids."""
    _, bad, message = next(c for c in ds.corrupted() if c[0] == "dlba_sum")
    y, x = ds.file_of("one_row", "dlba"), ds.file_of("v2_required", "dlba")
    T = lp.Col("timestamp")
    w = Walk(store, "seq_intern_order", "intern order")
    try:
        for buf in (y, x, bad):
            arr = np.frombuffer(buf, dtype=np.uint8)
            w.keep.append(arr)
            w.eng.put_parquet(w.table, arr, borrow=True)
        refused = m.Plan("refused", "agg", ("s",), (lp.Count(T),), T.GtEq(lp.Literal(1)))  # (prunes Y: one row, timestamp 0)
        for _ in range(2):
            with pytest.raises(_lib.FrostGPUError) as e:
                w.stats(refused)
            assert e.value.code == _lib.FGPU_ERR_UNSUPPORTED and "column s: " + message in e.value.msg, e.value.msg
        w.eng.drop_part(w.table, 2)
        q, _ = w._prepare(w.table, m.Plan("all", "agg", ("s",), (lp.Count(T),)))
        try:
            batches, _ = w._execute(w.table, q)
        finally:
            w.lib.fgpu_query_free(q)
        xs, ys = (ds.table("v2_required").column("s").to_pylist(), ds.table("one_row").column("s").to_pylist())
        assert not set(ys) & set(xs)
        assert w._dict("s") == ds.first_occurrence(xs) + ys
        exp = {}
        for v in ys + xs:
            exp[(v,)] = (exp.get((v,), (0,))[0] + 1,)
        assert ne.result_map([b for b in batches if b.num_rows], ["s"], [lp.Count(T)]) == exp
    finally:
        w.close()
