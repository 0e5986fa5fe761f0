"""DELTA_BINARY_PACKED int64 column chunks on the host, against pyarrow's read: `describe_parquet` unpacks every layout
of tests/delta_int64.py into the dense value array of a CK_PLAIN64 chunk, a required layout's image is as large as its
PLAIN twin's, a page that breaks one validation rule is refused with its own message while the file's other column
describes, and the layouts refused before keep their messages."""
import pytest

from frostdb_b200 import _lib
from frostdb_b200 import dynparquet as dp
from tests import delta_int64 as di


@pytest.mark.parametrize("name", di.NAMES)
def test_layout_is_what_it_says(name):
    for col in ("timestamp", "value"):
        assert all(e == {di.DBP} for e in di.encodings(di.file_of(name), col)), col
        assert all(e == {"PLAIN"} for e in di.encodings(di.twin_of(name), col)), col


def _check_describe(buf, exp: dict):
    d = _lib.describe_parquet(buf)
    slices = di.row_group_slices(buf)
    assert [rg["n_rows"] for rg in d["row_groups"]] == [e - b for b, e in slices]
    for g, (b, e) in enumerate(slices):
        for col, values in exp.items():
            c = d["row_groups"][g]["columns"][col]
            assert "error" not in c, (g, col, c["error"])
            assert c["kind"] == di.CK_PLAIN64
            assert c["decoded"] == values[b:e], (g, col)
            assert c["tile_index_ok"], (g, col)
            assert c["n_values"] == sum(v is not None for v in values[b:e])
    return d


@pytest.mark.parametrize("name", di.NAMES)
def test_describe_decodes_like_pyarrow(name):
    t = dp.read_part(di.twin_of(name))
    exp = {col: t.column(col).to_pylist() for col in ("timestamp", "value")}
    d = _check_describe(di.file_of(name), exp)
    if not di.LAYOUT_BY_NAME[name].nullable:
        assert d["image_bytes"] == _lib.describe_parquet(di.twin_of(name))["image_bytes"]


@pytest.mark.parametrize("name,buf,exp", di.hand_layouts(), ids=[c[0] for c in di.hand_layouts()])
def test_hand_assembled_pages(name, buf, exp):
    _check_describe(buf, {"value": exp, "timestamp": list(range(len(exp)))})


@pytest.mark.parametrize("name,buf,message", di.corrupted(), ids=[c[0] for c in di.corrupted()])
def test_corrupted_page_is_refused(name, buf, message):
    d = _lib.describe_parquet(buf)
    c = d["row_groups"][0]["columns"]
    assert c["value"].get("error") == message, c["value"]
    assert c["timestamp"]["decoded"] == list(range(d["row_groups"][0]["n_rows"]))


def test_corrupted_messages_are_distinct_per_rule():
    by_rule = {}
    for name, _, message in di.corrupted():
        by_rule.setdefault(message, []).append(name)
    assert len(by_rule) == 5, by_rule  # block size, miniblock size, count, bit width, overrun (header, widths, miniblock)


def test_layouts_refused_before_keep_their_messages():
    assert _lib.describe_parquet(di.double_delta())["row_groups"][0]["columns"]["value"] == {"error": "unsupported page encoding 5"}
    c = _lib.describe_parquet(di.dictionary_then_delta())["row_groups"][0]["columns"]
    assert c["value"] == {"error": "column chunk mixes dictionary and PLAIN pages"}
    assert "error" not in c["timestamp"]


def test_schema_encoding_writes_what_it_claims():
    cols = di.columns("sorted")
    buf = dp.write_part(di.schema(cols, delta=True), cols, sort=False, row_group_size=4096)
    for col in ("timestamp", "value"):
        assert all(e == {di.DBP} for e in di.encodings(buf, col))
    assert all(e == {"RLE_DICTIONARY", "PLAIN"} or e == {"RLE_DICTIONARY"} for e in di.encodings(buf, "labels.a"))
    for typ, col in ((dp.TYPE_STRING, "stacktrace"), (dp.TYPE_DOUBLE, "floatvalue")):
        s = dp.SampleDefinitionWithFloat()
        for c in s.columns:
            if c.name == col:
                c.delta_binary_packed = True
        with pytest.raises(ValueError, match="DELTA_BINARY_PACKED"):
            dp.write_part(s, dict(cols, floatvalue=[0.5] * len(cols["timestamp"])), sort=False)
