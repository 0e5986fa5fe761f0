"""ctypes binding of libfrostgpu.so (include/frostgpu.h).

The library is the product; there is no Python or CPU implementation behind it.  Loading fails
loudly when the shared object has not been built (run `python __graft_entry__.py` or
`make -C frostdb_b200/csrc`).
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libfrostgpu.so")

FGPU_OK = 0
FGPU_ERR_INVALID = -1
FGPU_ERR_PARQUET = -2
FGPU_ERR_UNSUPPORTED = -3
FGPU_ERR_CUDA = -4
FGPU_ERR_NOT_FOUND = -5
FGPU_ERR_OOM = -6
FGPU_ERR_NO_DEVICE = -7
FGPU_ERR_END = -8

ABI_VERSION = 1

# logicalplan.Op (query/logicalplan/expr.go:13-33)
OP_EQ, OP_NOT_EQ, OP_LT, OP_LT_EQ, OP_GT, OP_GT_EQ = 1, 2, 3, 4, 5, 6
OP_REGEX_MATCH, OP_REGEX_NOT_MATCH, OP_AND, OP_OR = 7, 8, 9, 10
OP_ADD, OP_SUB, OP_MUL, OP_DIV, OP_CONTAINS, OP_NOT_CONTAINS = 11, 12, 13, 14, 15, 16
# logicalplan.AggFunc (expr.go:718-729)
AGG_SUM, AGG_MIN, AGG_MAX, AGG_COUNT, AGG_AVG, AGG_UNIQUE, AGG_AND = 1, 2, 3, 4, 5, 6, 7

SCALAR_NULL, SCALAR_INT64, SCALAR_FLOAT64, SCALAR_STRING = 0, 1, 2, 3
EXPR_COLUMN, EXPR_DYNCOLUMN, EXPR_LITERAL, EXPR_BINARY = 1, 2, 3, 4
PLAN_AGGREGATE, PLAN_DISTINCT, PLAN_FILTER = 1, 2, 3
PUT_DEFAULT, PUT_BORROW_PINNED = 0, 1
COMM_HANDLE_BYTES = 128


class FrostGPUError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"libfrostgpu error {code}: {msg}")
        self.code = code
        self.msg = msg


class Config(C.Structure):
    _fields_ = [("abi_version", C.c_int32), ("device", C.c_int32), ("tile_rows", C.c_int32),
                ("flags", C.c_int32), ("staging_bytes", C.c_uint64)]


class Scalar(C.Structure):
    _fields_ = [("type", C.c_int32), ("_pad", C.c_int32), ("i64", C.c_int64), ("f64", C.c_double),
                ("bytes", C.c_void_p), ("len", C.c_uint64)]


MATCH_FN = C.CFUNCTYPE(C.c_int32, C.c_void_p, C.c_void_p, C.c_uint64)


class Expr(C.Structure):
    _fields_ = [("kind", C.c_int32), ("op", C.c_int32), ("left", C.c_int32), ("right", C.c_int32),
                ("name", C.c_char_p), ("literal", Scalar), ("match", MATCH_FN), ("match_user", C.c_void_p)]


class Agg(C.Structure):
    _fields_ = [("func", C.c_int32), ("expr", C.c_int32)]


class Plan(C.Structure):
    _fields_ = [("table", C.c_char_p), ("kind", C.c_int32), ("n_exprs", C.c_int32),
                ("exprs", C.POINTER(Expr)), ("filter", C.c_int32), ("n_group_by", C.c_int32),
                ("group_by", C.POINTER(C.c_int32)), ("n_aggs", C.c_int32), ("aggs", C.POINTER(Agg))]


class Stats(C.Structure):
    _fields_ = [("rows_scanned", C.c_uint64), ("rows_selected", C.c_uint64), ("groups", C.c_uint64),
                ("algorithmic_bytes", C.c_uint64), ("metadata_bytes", C.c_uint64),
                ("kernel_launches", C.c_uint32), ("row_groups", C.c_uint32),
                ("scan_kernel_ms", C.c_float), ("total_device_ms", C.c_float), ("h2d_ms", C.c_float),
                ("h2d_bytes", C.c_uint64), ("d2h_bytes", C.c_uint64),
                ("row_groups_pruned", C.c_uint32), ("row_groups_runs", C.c_uint32),
                ("row_groups_tiles", C.c_uint32), ("row_groups_prefix", C.c_uint32), ("rows_touched", C.c_uint64)]

    def asdict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


class ArrowSchema(C.Structure):
    pass


class ArrowArray(C.Structure):
    pass


ArrowSchema._fields_ = [("format", C.c_char_p), ("name", C.c_char_p), ("metadata", C.c_char_p),
                        ("flags", C.c_int64), ("n_children", C.c_int64),
                        ("children", C.POINTER(C.POINTER(ArrowSchema))),
                        ("dictionary", C.POINTER(ArrowSchema)), ("release", C.c_void_p),
                        ("private_data", C.c_void_p)]
ArrowArray._fields_ = [("length", C.c_int64), ("null_count", C.c_int64), ("offset", C.c_int64),
                       ("n_buffers", C.c_int64), ("n_children", C.c_int64),
                       ("buffers", C.POINTER(C.c_void_p)),
                       ("children", C.POINTER(C.POINTER(ArrowArray))),
                       ("dictionary", C.POINTER(ArrowArray)), ("release", C.c_void_p),
                       ("private_data", C.c_void_p)]

# Every symbol include/frostgpu.h declares, with its ctypes signature.
_SIGNATURES = {
    "fgpu_init": ([C.POINTER(Config), C.POINTER(C.c_void_p)], C.c_int32),
    "fgpu_shutdown": ([C.c_void_p], C.c_int32),
    "fgpu_last_error": ([], C.c_char_p),
    "fgpu_abi_version": ([], C.c_int32),
    "fgpu_part_put_parquet": ([C.c_void_p, C.c_char_p, C.c_uint64, C.c_uint64, C.c_void_p, C.c_uint64, C.c_int32], C.c_int32),
    "fgpu_part_put_arrow": ([C.c_void_p, C.c_char_p, C.c_uint64, C.c_uint64, C.c_void_p, C.c_void_p], C.c_int32),
    "fgpu_host_alloc": ([C.c_uint64, C.POINTER(C.c_void_p)], C.c_int32),
    "fgpu_host_free": ([C.c_void_p], C.c_int32),
    "fgpu_part_drop": ([C.c_void_p, C.c_char_p, C.c_uint64], C.c_int32),
    "fgpu_table_drop": ([C.c_void_p, C.c_char_p], C.c_int32),
    "fgpu_query_prepare": ([C.c_void_p, C.POINTER(Plan), C.POINTER(C.c_void_p)], C.c_int32),
    "fgpu_query_execute": ([C.c_void_p, C.c_void_p, C.c_uint64, C.POINTER(C.c_void_p)], C.c_int32),
    "fgpu_result_next": ([C.c_void_p, C.c_void_p, C.c_void_p], C.c_int32),
    "fgpu_result_stats": ([C.c_void_p, C.POINTER(Stats)], C.c_int32),
    "fgpu_result_free": ([C.c_void_p], C.c_int32),
    "fgpu_query_free": ([C.c_void_p], C.c_int32),
    "fgpu_dict_export": ([C.c_void_p, C.c_char_p, C.c_char_p, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64), C.POINTER(C.c_uint32)], C.c_int32),
    "fgpu_dict_preload": ([C.c_void_p, C.c_char_p, C.c_char_p, C.c_void_p, C.c_uint64, C.c_uint32], C.c_int32),
    "fgpu_parquet_dict_values": ([C.c_void_p, C.c_uint64, C.c_char_p, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64), C.POINTER(C.c_uint32)], C.c_int32),
    "fgpu_query_execute_partial": ([C.c_void_p, C.c_void_p, C.c_uint64, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.POINTER(C.c_uint64)], C.c_int32),
    "fgpu_result_merge_partials": ([C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_int32], C.c_int32),
    "fgpu_result_partial_is_additive": ([C.c_void_p, C.POINTER(C.c_int32)], C.c_int32),
    "fgpu_comm_export": ([C.c_void_p, C.c_int32, C.c_int32, C.c_uint64, C.c_void_p], C.c_int32),
    "fgpu_comm_open": ([C.c_void_p, C.c_void_p], C.c_int32),
    "fgpu_comm_close": ([C.c_void_p], C.c_int32),
    "fgpu_query_execute_collective": ([C.c_void_p, C.c_void_p, C.c_uint64, C.POINTER(C.c_void_p)], C.c_int32),
    "fgpu_query_execute_collective_begin": ([C.c_void_p, C.c_void_p, C.c_uint64, C.POINTER(C.c_void_p)], C.c_int32),
    "fgpu_query_execute_collective_end": ([C.c_void_p, C.c_void_p], C.c_int32),
    "fgpu_rowgroup_leaf_mode": ([C.c_int32, C.c_int64, C.c_int32, C.c_int64, C.c_int64, C.c_int64, C.c_int64, C.POINTER(C.c_int32)], C.c_int32),
    "fgpu_part_decode_column": ([C.c_void_p, C.c_char_p, C.c_uint64, C.c_char_p, C.c_void_p, C.c_void_p], C.c_int32),
    "fgpu_parquet_describe": ([C.c_void_p, C.c_uint64, C.c_int32, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64)], C.c_int32),
    "fgpu_xxhash64": ([C.c_char_p, C.c_uint64, C.c_uint64, C.POINTER(C.c_uint64)], C.c_int32),
    "fgpu_bloom_check": ([C.c_void_p, C.c_uint64, C.c_uint64, C.POINTER(C.c_int32)], C.c_int32),
    "fgpu_bloom_insert": ([C.c_void_p, C.c_uint64, C.c_uint64], C.c_int32),
    "fgpu_lz4_raw_inflate": ([C.c_char_p, C.c_uint64, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64)], C.c_int32),
    "fgpu_parquet_rowgroup_may_match_eq": ([C.c_char_p, C.c_uint64, C.c_int32, C.c_char_p, C.c_int32, C.c_int64, C.c_double, C.c_char_p, C.c_uint64,
                                            C.POINTER(C.c_int32)], C.c_int32),
}

_lib = None


def load() -> C.CDLL:
    """Loads libfrostgpu.so; raises if it is missing (no fallback of any kind)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise FileNotFoundError(
            f"{LIB_PATH} is not built. Build it with `make -C frostdb_b200/csrc` (or "
            "`python -c 'import __graft_entry__ as g; g.build()'`). frostdb_b200 has no CPU fallback.")
    lib = C.CDLL(LIB_PATH)
    for name, (argtypes, restype) in _SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if a declared symbol is not exported
        fn.argtypes = argtypes
        fn.restype = restype
    if lib.fgpu_abi_version() != ABI_VERSION:
        raise RuntimeError("libfrostgpu ABI version mismatch")
    _lib = lib
    return lib


def check(rc: int) -> None:
    if rc != FGPU_OK:
        raise FrostGPUError(rc, load().fgpu_last_error().decode("utf-8", "replace"))


def describe_parquet(buf: bytes, tile_rows: int = 0) -> dict:
    """Host-only: what fgpu_part_put_parquet would lay out for this file (no GPU needed)."""
    import json
    lib = load()
    n = C.c_uint64(0)
    src = (C.c_char * len(buf)).from_buffer_copy(buf)
    check(lib.fgpu_parquet_describe(C.addressof(src), len(buf), tile_rows, None, 0, C.byref(n)))
    out = C.create_string_buffer(n.value)
    check(lib.fgpu_parquet_describe(C.addressof(src), len(buf), tile_rows, C.addressof(out), n.value, C.byref(n)))
    return json.loads(out.raw[: n.value].decode("utf-8"))


def lz4_raw_inflate(block: bytes, size: int) -> bytes:
    """Host-only: one LZ4_RAW block that must inflate to exactly `size` bytes (FrostGPUError when it is refused)."""
    lib = load()
    out = C.create_string_buffer(max(size, 1))
    n = C.c_uint64(0)
    check(lib.fgpu_lz4_raw_inflate(block, len(block), C.addressof(out), size, C.byref(n)))
    return out.raw[:n.value]


def _parse_blob(raw: bytes, count: int):
    out, p = [], 0
    for _ in range(count):
        l = int.from_bytes(raw[p:p + 4], "little")
        out.append(raw[p + 4:p + 4 + l])
        p += 4 + l
    return out


def parquet_dict_values(buf, column: str):
    """Host-only: distinct dictionary entries of `column` in a Parquet file (bytes or numpy uint8 array)."""
    lib = load()
    if isinstance(buf, (bytes, bytearray, memoryview)):
        src = (C.c_char * len(buf)).from_buffer_copy(buf)
        addr, n = C.addressof(src), len(buf)
    else:
        addr, n = buf.ctypes.data, buf.nbytes
    ln, cnt = C.c_uint64(0), C.c_uint32(0)
    check(lib.fgpu_parquet_dict_values(addr, n, column.encode(), None, 0, C.byref(ln), C.byref(cnt)))
    out = C.create_string_buffer(max(ln.value, 1))
    check(lib.fgpu_parquet_dict_values(addr, n, column.encode(), C.addressof(out), ln.value, C.byref(ln), C.byref(cnt)))
    return _parse_blob(out.raw, cnt.value)
