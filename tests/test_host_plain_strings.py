"""PLAIN string column chunks on the host, against pyarrow's read: `describe_parquet` walks the length prefixes, interns
the values row by row and decodes every row of `s` as pyarrow does, as a dictionary chunk of the expected size;
`parquet_dict_values` lists the strings in the order a put interns them; malformed PLAIN pages are refused per chunk."""
import pytest

from frostdb_b200 import _lib
from tests import plain_strings as ps


@pytest.mark.parametrize("name", ps.NAMES)
def test_layout_is_what_it_says(name):
    layout = ps.LAYOUT_BY_NAME[name]
    for enc in ps.s_encodings(ps.file_of(name)):
        assert "PLAIN" in enc, enc
        assert ("RLE_DICTIONARY" in enc) == layout.fallback, enc
    for enc in ps.s_encodings(ps.twin_of(name)):
        assert "RLE_DICTIONARY" in enc, enc


@pytest.mark.parametrize("twin", [False, True])
@pytest.mark.parametrize("name", ps.NAMES)
def test_describe_decodes_like_pyarrow(name, twin):
    buf = ps.twin_of(name) if twin else ps.file_of(name)
    d = _lib.describe_parquet(buf)
    s = ps.table(name).column("s").to_pylist()
    slices = ps.row_group_slices(buf)
    assert [rg["n_rows"] for rg in d["row_groups"]] == [e - b for b, e in slices]
    for g, (b, e) in enumerate(slices):
        c = d["row_groups"][g]["columns"]["s"]
        assert "error" not in c, (g, c["error"])
        assert c["kind"] == ps.CK_DICT_STR
        assert c["decoded"] == s[b:e], g
        assert c["tile_index_ok"], g
        assert c["dict_size"] == len(ps.first_occurrence(s[b:e])), g
        assert c["n_values"] == sum(v is not None for v in s[b:e])
        for col in ("timestamp", "value", "fvalue"):
            assert c is not None and d["row_groups"][g]["columns"][col]["decoded"] == ps.table(name).column(col).to_pylist()[b:e]


@pytest.mark.parametrize("name", ps.NAMES)
def test_dict_values_in_order_of_first_occurrence(name):
    """Per row group the dictionary page, then the PLAIN values not in it in order of first occurrence: for these
    writers (the dictionary is built in order of first occurrence too) the file's order of first occurrence."""
    exp = [v.encode() for v in ps.first_occurrence(ps.table(name).column("s").to_pylist())]
    assert _lib.parquet_dict_values(ps.file_of(name), "s") == exp
    assert _lib.parquet_dict_values(ps.twin_of(name), "s") == exp


def _marked_file(version):
    """One PLAIN page whose last two values are MARKER_A, MARKER_B."""
    import io

    import pyarrow as pa
    import pyarrow.parquet as pq
    vals = [f"v{i}" for i in range(40)] + ["MARKER_A", "MARKER_B"]
    t = pa.table({"s": pa.array(vals, pa.string()), "timestamp": pa.array(range(len(vals)), pa.int64())})
    sink = io.BytesIO()
    pq.write_table(t, sink, compression="NONE", use_dictionary=False, data_page_version=version, store_schema=False)
    buf = bytearray(sink.getvalue())
    at = buf.find(b"\x08\x00\x00\x00MARKER_A")
    assert at > 0 and buf.find(b"\x08\x00\x00\x00MARKER_A", at + 1) < 0
    return buf, at


@pytest.mark.parametrize("version", ["1.0", "2.0"])
def test_length_prefix_past_the_page_is_refused(version):
    buf, at = _marked_file(version)
    buf[at:at + 4] = (1 << 20).to_bytes(4, "little")
    d = _lib.describe_parquet(bytes(buf))
    c = d["row_groups"][0]["columns"]
    assert "PLAIN string length prefix overruns its page" in c["s"]["error"]
    assert "error" not in c["timestamp"] and c["timestamp"]["decoded"] == list(range(42))
    with pytest.raises(_lib.FrostGPUError, match="overruns its page"):
        _lib.parquet_dict_values(bytes(buf), "s")


@pytest.mark.parametrize("version", ["1.0", "2.0"])
def test_page_short_of_its_values_is_refused(version):
    """MARKER_A's prefix swallows MARKER_B: the page then holds one value fewer than its levels say."""
    buf, at = _marked_file(version)
    buf[at:at + 4] = (8 + 4 + 8).to_bytes(4, "little")
    d = _lib.describe_parquet(bytes(buf))
    c = d["row_groups"][0]["columns"]
    assert "PLAIN string page shorter than its value count" in c["s"]["error"]
    assert "error" not in c["timestamp"]
    with pytest.raises(_lib.FrostGPUError, match="shorter than its value count"):
        _lib.parquet_dict_values(bytes(buf), "s")
