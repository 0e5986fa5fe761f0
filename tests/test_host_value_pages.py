"""The three ways a page's int64 values reach a chunk's dense value array (copied from the file, decoded from a
DELTA_BINARY_PACKED stream, inflated from an LZ4_RAW block), interleaved in one chunk's page list: `describe_parquet`
fills the holes the device would fill with the host's reference and decodes what pyarrow reads."""
import io

import pyarrow.parquet as pq

from frostdb_b200 import _lib
from tests import lz4_pages as lz


def test_describe_fills_every_kind_of_page_like_pyarrow():
    buf, exp = lz.mixed_fills()
    c = _lib.describe_parquet(buf)["row_groups"][0]["columns"]["value"]
    assert "error" not in c, c
    assert c["kind"] == lz.CK_PLAIN64 and c["codec"] == lz.CODEC_LZ4_RAW
    assert c["decoded"] == pq.read_table(io.BytesIO(buf)).column("value").to_pylist() == exp
    assert c["lz4_device_pages"] == 2
