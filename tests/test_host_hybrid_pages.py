"""The host half of the hybrid-stream decoder on the layout zoo of tests/hybrid_pages.py, against pyarrow's read:
`describe_parquet` (walk_hybrid, the run directories, the cursor seeds, the row-space directory, the padded tables)
decodes every column as pyarrow does, refuses the over-wide chunks, and builds the directories each layout implies;
the oracle decodes every column as pyarrow does and answers the zoo's aggregate plans like the numpy reference at 1
and 4 threads."""
import pytest

from frostdb_b200 import _lib
from frostdb_b200 import logicalplan as lp
from oracle.oracle import OracleTable
from tests import hybrid_pages as hp
from tests import numeric_edges as ne
from tests.oracle_scan import OracleEngine, OracleTableHandle, oracle_query

ZOO_COLUMNS = ("labels.z", "dictvalue")
NAMES = [l.name for l in hp.LAYOUTS]
HOST_DECODE_ROWS = 65536  # describe decodes row groups up to this size


def _slices(layout):
    out, s = [], 0
    for n in layout.rg_rows:
        out.append((s, s + n))
        s += n
    return out


@pytest.mark.parametrize("name", NAMES)
def test_describe_decodes_like_pyarrow(name):
    layout = hp.LAYOUT_BY_NAME[name]
    d = _lib.describe_parquet(hp.file_of(name))
    t = hp.read(name)
    assert [rg["n_rows"] for rg in d["row_groups"]] == layout.rg_rows
    for g, (s, e) in enumerate(_slices(layout)):
        cols = d["row_groups"][g]["columns"]
        for col in t.column_names:
            c = cols[col]
            if layout.error and col in ZOO_COLUMNS:
                assert layout.error in c.get("error", ""), (col, c)
                assert "decoded" not in c
                continue
            assert "error" not in c, (col, c["error"])
            if e - s <= HOST_DECODE_ROWS:
                assert c["decoded"] == t.column(col).to_pylist()[s:e], (g, col)
                assert c["tile_index_ok"], (g, col)
                assert c.get("row_runs_ok", True), (g, col)


@pytest.mark.parametrize("name", NAMES)
def test_directories_are_what_the_layout_implies(name):
    """n_runs of both zoo columns (unpacked short literals, runs merged within and across pages, 72-value literals and
    long bit-packed runs kept); the row-space directory of labels.z exactly where the layout is run-length only, with
    the stated run count, and runs long enough for the sorted-run kernel."""
    layout = hp.LAYOUT_BY_NAME[name]
    if layout.error:
        pytest.skip("refused layout: no directory")
    d = _lib.describe_parquet(hp.file_of(name))
    for g, rg in enumerate(d["row_groups"]):
        z, dv = rg["columns"]["labels.z"], rg["columns"]["dictvalue"]
        assert z["n_runs"] == dv["n_runs"] == layout.n_runs[g], (g, z["n_runs"], dv["n_runs"])
        if rg["n_rows"] > HOST_DECODE_ROWS:
            continue  # describe reports the row-space directory with the decode; the GPU tests assert its kernel
        if layout.sorted:
            assert z["n_row_runs"] == (layout.n_row_runs or layout.n_runs)[g], g
            assert z["n_row_runs"] * 32 <= rg["n_rows"] + 1024
        else:
            assert "n_row_runs" not in z, g  # bit-packed runs: no row-space directory


@pytest.mark.parametrize("name", NAMES)
def test_oracle_decodes_like_pyarrow(name):
    layout = hp.LAYOUT_BY_NAME[name]
    t = hp.read(name)
    ot = OracleTable()
    try:
        ot.add_parquet(hp.file_of(name))
        for g, (s, e) in enumerate(_slices(layout)):
            for col in t.column_names:
                assert ot.decode_column(0, g, col) == t.column(col).to_pylist()[s:e], (g, col)
    finally:
        ot.close()


@pytest.mark.parametrize("threads", [1, 4])
@pytest.mark.parametrize("name", [n for n in NAMES if max(hp.LAYOUT_BY_NAME[n].rg_rows) <= HOST_DECODE_ROWS])
def test_oracle_aggregates_like_the_reference(name, threads):
    layout = hp.LAYOUT_BY_NAME[name]
    ref = hp.Reference(name)
    eng = OracleEngine(threads=threads)
    try:
        OracleTableHandle(eng, "zoo", hp.schema()).InsertParquet(hp.file_of(name))
        for filt, keys, aggs in hp.plans(layout):
            out = []
            q = oracle_query(eng, "zoo")
            q = q.Filter(filt) if filt is not None else q
            q.Aggregate(aggs, [lp.Col(k) for k in keys]).Execute(None, lambda c, r: out.append(r))
            what = f"{name} threads={threads} filter {filt.Name() if filt is not None else None} {keys}"
            ne.assert_same_result(ne.result_map(out, keys, aggs), ref.aggregate(filt, keys, aggs), aggs, what)
    finally:
        eng.close()
