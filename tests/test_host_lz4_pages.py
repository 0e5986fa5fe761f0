"""LZ4_RAW-compressed column chunks on the host, against pyarrow's read: `describe_parquet` inflates every layout of
tests/lz4_pages.py into what its uncompressed twin gives, a REQUIRED layout's image is as large as its twin's, the pages
the device would inflate follow the split rule (PLAIN INT64 / DOUBLE pages whose block holds nothing but values), the
host's block parser takes exactly the hand-assembled blocks pyarrow takes and inflates them to pyarrow's bytes, every
malformed block is refused with its own message while the file's other column still describes, and every other codec
keeps its refusal."""
import pytest

from frostdb_b200 import _lib
from frostdb_b200 import dynparquet as dp
from tests import delta_int64 as di
from tests import lz4_pages as lz

COLS = ("timestamp", "value")


@pytest.mark.parametrize("name", lz.NAMES)
def test_layout_is_what_it_says(name):
    assert all(c == {"LZ4"} for c in lz.codecs(lz.file_of(name)).values())
    assert all(c == {"UNCOMPRESSED"} for c in lz.codecs(lz.twin_of(name)).values())
    enc = {di.DBP} if lz.LAYOUT_BY_NAME[name].delta else {"PLAIN"}
    for col in COLS:
        assert all(e == enc for e in di.encodings(lz.file_of(name), col)), col


@pytest.mark.parametrize("name", lz.NAMES)
def test_describe_equals_pyarrow_and_the_twin(name):
    l = lz.LAYOUT_BY_NAME[name]
    t = dp.read_part(lz.twin_of(name))
    d, twin = _lib.describe_parquet(lz.file_of(name)), _lib.describe_parquet(lz.twin_of(name))
    slices = di.row_group_slices(lz.file_of(name))
    v1 = l.version == "1.0"
    device_pages = {col: 0 for col in COLS}
    for g, (b, e) in enumerate(slices):
        for col in d["row_groups"][g]["columns"]:
            c, tc = d["row_groups"][g]["columns"][col], twin["row_groups"][g]["columns"][col]
            assert "error" not in c, (g, col, c)
            assert c["decoded"] == tc["decoded"], (g, col)
            assert c["codec"] == lz.CODEC_LZ4_RAW and "codec" not in tc
            if col in COLS:
                assert c["decoded"] == t.column(col).to_pylist()[b:e], (g, col)
                assert c["kind"] == lz.CK_PLAIN64
                device_pages[col] += c["lz4_device_pages"]
            else:
                assert c["lz4_device_pages"] == 0, (g, col)
    # the split rule: PLAIN values of v2 pages, and of v1 pages of a REQUIRED column, are inflated on the device (pyarrow
    # stores a v2 page's values uncompressed when LZ4 does not shrink them: those are read as they are)
    for col in COLS:
        device = not l.delta and not (v1 and l.nullable and col == "value")
        assert (device_pages[col] > 0) == device, (col, device_pages)
    if not l.nullable:
        assert d["image_bytes"] == twin["image_bytes"]


@pytest.mark.parametrize("name", lz.NAMES[:2])
def test_stored_bytes_are_the_inflated_bytes(name):
    d = _lib.describe_parquet(lz.file_of(name))
    for col in COLS:
        comp, raw = lz.footer_sizes(lz.file_of(name), col)
        assert sum(rg["columns"][col]["stored_bytes"] for rg in d["row_groups"]) == raw > comp, col
    twin = _lib.describe_parquet(lz.twin_of(name))
    assert sum(rg["columns"]["value"]["stored_bytes"] for rg in twin["row_groups"]) == lz.footer_sizes(lz.twin_of(name), "value")[0]


@pytest.mark.parametrize("name", lz.STR_NAMES)
def test_string_layouts_describe_like_the_twin(name):
    d, twin = _lib.describe_parquet(lz.str_file_of(name)), _lib.describe_parquet(lz.str_twin_of(name))
    t = lz.str_table(name)
    b = 0
    for g, (rg, trg) in enumerate(zip(d["row_groups"], twin["row_groups"])):
        for col, c in rg["columns"].items():
            assert "error" not in c, (g, col, c)
            assert c["decoded"] == trg["columns"][col]["decoded"], (g, col)
            if col == "s":
                assert c["lz4_device_pages"] == 0
        assert rg["columns"]["s"]["decoded"] == t.column("s").to_pylist()[b:b + rg["n_rows"]]
        b += rg["n_rows"]


@pytest.mark.parametrize("name", lz.STR_NAMES)
def test_dict_values_equal_the_twins(name):
    assert _lib.parquet_dict_values(lz.str_file_of(name), "s") == _lib.parquet_dict_values(lz.str_twin_of(name), "s")


@pytest.mark.parametrize("name,block,data", lz.valid_blocks(), ids=[b[0] for b in lz.valid_blocks()])
def test_parser_takes_what_pyarrow_takes(name, block, data):
    assert lz.pyarrow_accepts(block, len(data))
    assert _lib.lz4_raw_inflate(block, len(data)) == lz.LZ4.decompress(block, decompressed_size=len(data), asbytes=True) == data


@pytest.mark.parametrize("name,block,size,message", lz.malformed(), ids=[m[0] for m in lz.malformed()])
def test_malformed_block_is_refused_with_its_message(name, block, size, message):
    with pytest.raises(_lib.FrostGPUError) as e:
        _lib.lz4_raw_inflate(block, size)
    assert e.value.msg == message and e.value.code == _lib.FGPU_ERR_PARQUET
    assert lz.pyarrow_accepts(block, size) == (name in lz.PYARROW_TAKES)


def test_malformed_messages_are_distinct():
    messages = [m[3] for m in lz.malformed()]
    assert len(set(messages)) == len(messages)


def test_empty_values_region():
    """An empty output is the block 0x00 for the parser (pyarrow refuses 0 stored bytes as a block); a page's empty
    values region may be either (v2_empty_values_0_bytes)."""
    assert _lib.lz4_raw_inflate(b"\x00", 0) == b""
    assert not lz.pyarrow_accepts(b"", 0)
    with pytest.raises(_lib.FrostGPUError, match="empty"):
        _lib.lz4_raw_inflate(b"", 0)


@pytest.mark.parametrize("name,buf,exp,device", lz.hand_layouts(), ids=[h[0] for h in lz.hand_layouts()])
def test_hand_assembled_pages(name, buf, exp, device):
    rg = _lib.describe_parquet(buf)["row_groups"][0]
    c = rg["columns"]["value"]
    assert "error" not in c, c
    assert c["lz4_device_pages"] == device
    if rg["n_rows"] <= 65536:  # (describe decodes small row groups only)
        assert c["decoded"] == exp
        assert rg["columns"]["timestamp"]["decoded"] == list(range(len(exp)))


@pytest.mark.parametrize("name,buf,message", lz.corrupted_files(), ids=[c[0] for c in lz.corrupted_files()])
def test_corrupted_page_is_refused_and_the_other_column_describes(name, buf, message):
    rg = _lib.describe_parquet(buf)["row_groups"][0]
    assert rg["columns"]["value"] == {"error": message}
    assert rg["columns"]["timestamp"]["decoded"] == list(range(rg["n_rows"]))


@pytest.mark.parametrize("codec", [1, 2, 4, 5, 6, 3])
def test_other_codecs_keep_their_refusal(codec):
    """SNAPPY, GZIP, BROTLI, LZ4 (Hadoop framing), ZSTD and LZO."""
    c = _lib.describe_parquet(lz.codec_file(codec))["row_groups"][0]["columns"]
    assert c["value"] == {"error": f"compressed column chunk (codec {codec}) is not supported"}
    assert "error" not in c["timestamp"]


def test_default_compression_writes_the_same_bytes():
    cols = lz.columns("sorted")
    s = di.schema(cols, delta=False)
    assert all(c.compression == "NONE" for c in s.columns)
    assert dp.write_part(s, cols, sort=False) == dp.write_part(lz.schema("sorted", lz4=False), cols, sort=False)
    with pytest.raises(ValueError, match="compression"):
        s.columns[0].compression = "SNAPPY"
        dp.write_part(s, cols, sort=False)
