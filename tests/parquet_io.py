"""ctypes helpers around the Parquet writer shared by the GPU tests and tools/parquet_measure.py: the columns of an
Arrow emit's host image as tests/parquet_ref.py columns, the field list the tests use, the three write calls, the file
bytes (from the host image or device memory) and the metrics."""
import ctypes as C

import numpy as np

import parquet_ref as R
from etl_b200 import abi


def _buf(ptr, n, dtype):
    return np.frombuffer((C.c_uint8 * (n * np.dtype(dtype).itemsize)).from_address(ptr), dtype=dtype).copy() if n else np.zeros(0, dtype)


def _bits(ptr, n):
    if not n:
        return np.zeros(0, bool)
    raw = np.frombuffer((C.c_uint8 * ((n + 7) // 8)).from_address(ptr), dtype=np.uint8)
    return np.unpackbits(raw, bitorder="little")[:n].astype(bool)


def _column(col, n):
    t = col.arrow_type
    out = {"type": t, "valid": _bits(col.validity, n)}
    if t == R.BOOLEAN:
        out["values"] = _bits(col.values, n)
    elif t == R.UUID:
        out["values"] = _buf(col.values, n * 16, np.uint8).reshape(n, 16)
    elif t in R.NP:
        out["values"] = _buf(col.values, n, R.NP[t])
    elif t in (R.UTF8, R.LARGE_BINARY):
        out["offsets"] = _buf(col.offsets, n + 1, "<i4" if t == R.UTF8 else "<i8").astype(np.int64) if n else np.zeros(1, np.int64)
        out["data"] = bytes((C.c_uint8 * col.data_bytes).from_address(col.data)) if col.data_bytes else b""
    return out


def emit_columns(lib, a):
    """the emit's columns from its host image, as parquet_ref columns"""
    n = lib.etl_dec_arrow_rows(a)
    cols = []
    for c in range(lib.etl_dec_arrow_cols(a)):
        col = abi.ArrowColumn()
        assert lib.etl_dec_arrow_column(a, c, 1, C.byref(col)) == 0
        if col.arrow_type != R.LIST:
            cols.append(_column(col, n))
            continue
        kid, ne = abi.ArrowColumn(), C.c_uint64()
        assert lib.etl_dec_arrow_list_child(a, c, 1, C.byref(kid), C.byref(ne)) == 0
        cols.append({"type": R.LIST, "valid": _bits(col.validity, n),
                     "offsets": _buf(col.offsets, n + 1, "<i4").astype(np.int64) if n else np.zeros(1, np.int64),
                     "child": _column(kid, ne.value)})
    return cols


def fields_for(cols, required=()):
    """c<i> names, field ids 1.., element ids 1000.., the two CDC columns and the listed columns required"""
    n = len(cols)
    return [(f"c{i}" if i < n - 2 else ("cdc_operation", "sequence_number")[i - n + 2], i + 1, 1000 + i,
             1 if (i >= n - 2 or i in required) else 0) for i in range(n)]


def _arrays(fields, bloom):
    """the etl_parquet_field array of fields [(name as str or bytes, field_id, element_field_id, required)] and the
    etl_parquet_bloom array of bloom [(fpp, ndv, max_bytes)] (None: a NULL array)"""
    arr = (abi.ParquetField * max(1, len(fields)))()
    for i, f in enumerate(fields):
        arr[i].name = f[0].encode() if isinstance(f[0], str) else f[0]
        arr[i].field_id, arr[i].element_field_id, arr[i].required = f[1], f[2], f[3]
    barr = None
    if bloom is not None:
        barr = (abi.ParquetBloom * max(1, len(bloom)))()
        for i, (fpp, ndv, mb) in enumerate(bloom):
            barr[i].fpp, barr[i].ndv, barr[i].max_bytes = fpp, ndv, mb
    return arr, barr


def pq_write(lib, a, fields, rb, re, codec, to_host=1):
    arr, _ = _arrays(fields, None)
    h = C.c_void_p()
    rc = lib.etl_dec_parquet_write(a, arr, len(fields), rb, re, codec, to_host, C.byref(h))
    return rc, h


def pq_write_bloom(lib, a, fields, bloom, rb, re, codec, to_host=1):
    """etl_dec_parquet_write_bloom; bloom: [(fpp, ndv, max_bytes)] or None (a NULL array)"""
    arr, barr = _arrays(fields, bloom)
    h = C.c_void_p()
    rc = lib.etl_dec_parquet_write_bloom(a, arr, barr, len(fields), rb, re, codec, to_host, C.byref(h))
    return rc, h


def write_files(lib, a, fields, bloom, ro, codec, to_host=1):
    """etl_dec_parquet_write_files over row offsets ro (len(ro) - 1 files); bloom: [(fpp, ndv, max_bytes)] or None"""
    arr, barr = _arrays(fields, bloom)
    offs = (C.c_uint64 * max(1, len(ro)))(*[int(x) for x in ro])
    h = C.c_void_p()
    rc = lib.etl_dec_parquet_write_files(a, arr, barr, len(fields), offs, max(0, len(ro) - 1), codec, to_host, C.byref(h))
    return rc, h


def _cudart():
    rt = C.CDLL("libcudart.so.12")
    rt.cudaMemcpy.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int]
    return rt


def device_bytes(ptr, n):
    """n bytes of device memory at ptr"""
    buf = C.create_string_buffer(max(1, n))
    if n:
        assert _cudart().cudaMemcpy(buf, ptr, n, 2) == 0                    # cudaMemcpyDeviceToHost
    return buf.raw[:n]


def file_bytes(lib, h):
    n = lib.etl_dec_parquet_size(h)
    return bytes((C.c_uint8 * n).from_address(lib.etl_dec_parquet_bytes(h, 1))) if n else b""


def metrics(lib, h, n_leaves):
    out = []
    for l in range(n_leaves):
        m = abi.ParquetMetrics()
        assert lib.etl_dec_parquet_metrics(h, l, C.byref(m)) == 0
        has = bool(m.flags & abi.PQ_HAS_MIN_MAX)
        out.append(dict(field_id=m.field_id, num_values=m.num_values, null_count=m.null_count, nan_count=m.nan_count,
                        compressed_bytes=m.compressed_bytes, uncompressed_bytes=m.uncompressed_bytes,
                        min=bytes((C.c_uint8 * m.min_len).from_address(m.min)) if has else None,
                        max=bytes((C.c_uint8 * m.max_len).from_address(m.max)) if has else None))
    return out
