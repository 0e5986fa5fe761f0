"""DELTA_LENGTH_BYTE_ARRAY and DELTA_BYTE_ARRAY string column chunks on the host, against pyarrow's read:
`describe_parquet` decodes the length streams, rebuilds the front-coded values and decodes every row of `s` as pyarrow
does, as a dictionary chunk of the expected size; `parquet_dict_values` lists the strings in the order a put interns
them; a page that breaks one validation rule is refused with its own message while the file's other column describes."""
import pytest

from frostdb_b200 import _lib
from tests import delta_strings as ds


@pytest.mark.parametrize("name,enc", ds.CASES, ids=ds.CASE_IDS)
def test_layout_is_what_it_says(name, enc):
    for e in ds.s_encodings(ds.file_of(name, enc)):
        assert ds.ENCODINGS[enc] in e and "PLAIN" not in e and "RLE_DICTIONARY" not in e, e
    for e in ds.s_encodings(ds.twin_of(name)):
        assert "RLE_DICTIONARY" in e, e
    for e in ds.s_encodings(ds.plain_of(name)):
        assert "PLAIN" in e and "RLE_DICTIONARY" not in e, e


def _check_describe(buf, s):
    d = _lib.describe_parquet(buf)
    slices = ds.row_group_slices(buf)
    assert [rg["n_rows"] for rg in d["row_groups"]] == [e - b for b, e in slices]
    for g, (b, e) in enumerate(slices):
        c = d["row_groups"][g]["columns"]["s"]
        assert "error" not in c, (g, c["error"])
        assert c["kind"] == ds.CK_DICT_STR
        if "decoded" in c:
            assert c["decoded"] == s[b:e], g
            assert c["tile_index_ok"], g
        assert c["dict_size"] == len(ds.first_occurrence(s[b:e])), g
        assert c["n_values"] == sum(v is not None for v in s[b:e])
    return d


@pytest.mark.parametrize("name,enc", ds.CASES, ids=ds.CASE_IDS)
def test_describe_decodes_like_pyarrow(name, enc):
    buf = ds.file_of(name, enc)
    t = ds.table(name)
    d = _check_describe(buf, t.column("s").to_pylist())
    for g, (b, e) in enumerate(ds.row_group_slices(buf)):
        for col in ("timestamp", "value", "fvalue"):
            assert d["row_groups"][g]["columns"][col]["decoded"] == t.column(col).to_pylist()[b:e]


@pytest.mark.parametrize("name,enc", ds.CASES, ids=ds.CASE_IDS)
def test_dict_values_in_order_of_first_occurrence(name, enc):
    exp = [v.encode() for v in ds.first_occurrence(ds.table(name).column("s").to_pylist())]
    assert _lib.parquet_dict_values(ds.file_of(name, enc), "s") == exp
    assert _lib.parquet_dict_values(ds.plain_of(name), "s") == exp
    assert _lib.parquet_dict_values(ds.twin_of(name), "s") == exp


def test_dictionary_pages_followed_by_delta_and_plain_pages():
    """The dictionary page's entries first, then the values of the DLBA, DBA and PLAIN pages not among them."""
    buf = ds.mixed_file()
    s = ds.mixed_strings()
    assert ds.s_encodings(buf) == [{"PLAIN", "RLE", "RLE_DICTIONARY", "DELTA_LENGTH_BYTE_ARRAY", "DELTA_BYTE_ARRAY"}]
    _check_describe(buf, s)
    dict_vals = [f"dict/{i:03d}" for i in range(20)]
    exp = dict_vals + [v for v in ds.first_occurrence(s) if v not in dict_vals]
    assert _lib.parquet_dict_values(buf, "s") == [v.encode() for v in exp]


@pytest.mark.parametrize("name,buf,message", ds.corrupted(), ids=[c[0] for c in ds.corrupted()])
def test_corrupted_page_is_refused(name, buf, message):
    d = _lib.describe_parquet(buf)
    c = d["row_groups"][0]["columns"]
    assert c["s"].get("error") == message, c["s"]
    assert "error" not in c["timestamp"]
    if "decoded" in c["timestamp"]:
        assert c["timestamp"]["decoded"] == list(range(d["row_groups"][0]["n_rows"]))
    with pytest.raises(_lib.FrostGPUError) as e:
        _lib.parquet_dict_values(buf, "s")
    assert message in str(e.value)


def test_corrupted_messages_are_distinct():
    msgs = [m for n, _, m in ds.corrupted() if n != "long_prefix"]
    assert len(set(msgs)) == len(msgs)
