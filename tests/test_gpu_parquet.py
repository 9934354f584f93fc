"""Parquet writer (csrc/parquet_write.cu) against the Python restatement of the file (tests/parquet_ref.py) fed the same
Arrow emit's columns: the uncompressed file byte for byte, the Snappy file page by page (headers equal except
compressed_page_size, payloads equal after pyarrow's Snappy, footer equal except sizes and offsets), the metrics, and
pyarrow's reading of the Snappy file against the emit.  Inputs: c1–c5, a COPY batch, a hand-built stream of every
column type with lists and float corners, long text across the 1 MiB page cut, more than 20 000 rows, a COPY table of
two row groups, required columns, row slices and zero rows; then the required-null report, the argument checks and
write/free cycles."""
import ctypes as C
import io
import math
import struct

import numpy as np
import pytest

import parquet_ref as R
import scenarios as sc
from parquet_io import emit_columns, fields_for, file_bytes, metrics, pq_write
from etl_b200 import abi, pgoutput as pg, workloads as wl
from test_gpu_arrow_copy import copy_batch
from test_gpu_copy import synth_rows
from test_gpu_rowbinary import hand_built

pytestmark = pytest.mark.gpu

ERR_INVALID_ARG = 1
EMIT_KINDS = 7 | abi.ARROW_ALL_COLUMNS | abi.ARROW_CDC_COLUMNS
INT4, TEXT = 23, 25


@pytest.fixture(scope="module")
def gpu():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from etl_b200 import decoder
    return decoder


# ------------------------------------------------------------------------------------------------ pyarrow comparison
def _norm_ref(col, n=None):
    t = col["type"]
    n = len(col["valid"]) if n is None else n
    if t == R.LIST:
        kid = _norm_ref(col["child"])
        o = col["offsets"]
        return [kid[o[i]:o[i + 1]] if col["valid"][i] else None for i in range(n)]
    out = []
    for i in range(n):
        if not col["valid"][i]:
            out.append(None)
        elif t == R.BOOLEAN:
            out.append(bool(col["values"][i]))
        elif t in (R.UTF8, R.LARGE_BINARY):
            out.append(col["data"][col["offsets"][i]:col["offsets"][i + 1]])
        elif t == R.UUID:
            out.append(bytes(col["values"][i]))
        elif t in (R.FLOAT32, R.FLOAT64):
            x = float(col["values"][i])
            out.append("nan" if math.isnan(x) else struct.pack("<d", x))
        else:
            out.append(int(col["values"][i]))
    return out


def _norm_pa(arr):
    import pyarrow as pa
    t = arr.type
    if isinstance(t, pa.BaseExtensionType):
        return _norm_pa(arr.storage)
    if pa.types.is_list(t) or pa.types.is_large_list(t):
        kid = _norm_pa(arr.values)
        o, v = arr.offsets.to_numpy(), arr.is_valid().to_numpy(zero_copy_only=False)
        return [kid[o[i]:o[i + 1]] if v[i] else None for i in range(len(arr))]
    if pa.types.is_string(t) or pa.types.is_large_string(t):
        arr = arr.cast(pa.large_binary())
    elif pa.types.is_date32(t):
        arr = arr.view(pa.int32())
    elif pa.types.is_timestamp(t) or pa.types.is_time64(t):
        arr = arr.view(pa.int64())
    vals = arr.to_pylist()
    if pa.types.is_floating(t):
        return [None if x is None else ("nan" if math.isnan(x) else struct.pack("<d", x)) for x in vals]
    return vals


def check_pyarrow(data, cols, fields, rb, re):
    import pyarrow.parquet as pq
    tab = pq.read_table(io.BytesIO(data))
    assert tab.num_rows == re - rb
    for i, (col, f) in enumerate(zip(cols, fields)):
        got = _norm_pa(tab.column(i).combine_chunks())
        want = _norm_ref(col)[rb:re]
        assert got == want, f"column {f[0]}"
        field = tab.schema.field(i)
        assert field.metadata[b"PARQUET:field_id"] == str(f[1]).encode()


# ------------------------------------------------------------------------------------------------ the check
MASK_CMD = {6, 7, 9}          # ColumnMetaData sizes and data_page_offset
MASK_RG = {2, 5, 6}           # RowGroup total_byte_size, file_offset, total_compressed_size


def _masked_footer(fm):
    fm = dict(fm)
    rgs = []
    for rg in fm.get(4, []):
        rg = {k: v for k, v in rg.items() if k not in MASK_RG}
        rg[1] = [{2: None, 3: {k: v for k, v in cc[3].items() if k not in MASK_CMD | {4}}} for cc in rg[1]]
        rgs.append(rg)
    fm[4] = rgs
    return fm


def check_write(lib, a, cols, fields, rb, re, what, cdc_ratio=False):
    want, want_m, want_pages = R.write(cols, fields, rb, re)
    rc, h = pq_write(lib, a, fields, rb, re, abi.PQ_UNCOMPRESSED)
    assert rc == 0, what
    got = file_bytes(lib, h)
    if got != want:
        at = next((i for i in range(min(len(got), len(want))) if got[i] != want[i]), min(len(got), len(want)))
        raise AssertionError(f"{what}: uncompressed file differs at byte {at} of {len(want)} (got {len(got)})")
    assert metrics(lib, h, len(fields)) == want_m, what
    lib.etl_dec_parquet_free(h)
    import pyarrow as pa
    snappy = pa.Codec("snappy")
    rc, h = pq_write(lib, a, fields, rb, re, abi.PQ_SNAPPY)
    assert rc == 0, what
    data = file_bytes(lib, h)
    pages = R.walk_pages(data)
    assert len(pages) == len(want_pages), what
    csize, usize = {}, {}
    for (ci, hd, hb, payload), (wci, whb, wpayload) in zip(pages, want_pages):
        wh, _ = R.read_struct(whb)
        assert ci == wci and {k: v for k, v in hd.items() if k != 3} == {k: v for k, v in wh.items() if k != 3}, what
        assert snappy.decompress(payload, decompressed_size=len(wpayload)).to_pybytes() == wpayload, what
        csize[ci] = csize.get(ci, 0) + len(hb) + len(payload)
        usize[ci] = usize.get(ci, 0) + len(hb) + len(wpayload)    # the header holds the compressed size: its width varies
    fm, _ = R.file_footer(data)
    wfm, _ = R.file_footer(want)
    assert _masked_footer(fm) == _masked_footer(wfm), what
    assert all(cc[3][4] == 1 for rg in fm.get(4, []) for cc in rg[1])
    got_m = metrics(lib, h, len(fields))
    sizes = ("compressed_bytes", "uncompressed_bytes")
    for g, w in zip(got_m, want_m):
        assert {k: v for k, v in g.items() if k not in sizes} == {k: v for k, v in w.items() if k not in sizes}, what
    for key, per_chunk in zip(sizes, (csize, usize)):
        assert [m[key] for m in got_m] == [sum(per_chunk.get(ci, 0) for ci in range(l, len(per_chunk), len(fields)))
                                           for l in range(len(fields))], (what, key)
    if cdc_ratio:
        for m in got_m[-2:]:
            assert m["compressed_bytes"] * 4 <= m["uncompressed_bytes"], (what, m)
    check_pyarrow(data, cols, fields, rb, re)
    lib.etl_dec_parquet_free(h)


def _decode_stream(gpu, tables, raw):
    dec = gpu.Decoder(0)
    for tid, cols in tables.items():
        dec.put_table_schema(tid, cols)
    st = gpu.Stager(len(raw) + 64, 2048)
    st.append_framed(raw)
    return dec, st


def _emit(lib, bh, si):
    a = C.c_void_p()
    assert lib.etl_dec_arrow_emit(bh._h, si, EMIT_KINDS, 1, C.byref(a)) == 0
    return a


def run_stream(gpu, tables, raw, what, slices=True, required=()):
    lib = abi.load()
    dec, st = _decode_stream(gpu, tables, raw)
    n_total = 0
    with dec.decode_input(st.view(), to_host=True) as bh:
        for si in range(len(bh.schemas())):
            a = _emit(lib, bh, si)
            cols = emit_columns(lib, a)
            n = lib.etl_dec_arrow_rows(a)
            fields = fields_for(cols, required)
            check_write(lib, a, cols, fields, 0, n, f"{what} v{si}", cdc_ratio=n >= 2000)
            if slices and n > 2:
                check_write(lib, a, cols, fields, n // 3, n - n // 4, f"{what} v{si} slice")
                check_write(lib, a, cols, fields, n // 2, n // 2, f"{what} v{si} empty")
            n_total += n
            lib.etl_dec_arrow_free(a)
    st.close()
    dec.close()
    return n_total


@pytest.mark.parametrize("name,scale", [("c1", 0.01), ("c2", 0.0005), ("c3", 0.001), ("c4", 0.002), ("c5", 0.0005)])
def test_workloads(gpu, name, scale):
    w = wl.make(name, scale, n_segments=1)
    stream, _ = w.generate()
    assert run_stream(gpu, w.table_schemas(), stream.tobytes(), name) > 0


def test_hand_built_every_type(gpu, oracle_mod):
    """every scalar type and List child type with NULLs, empty lists and NULL elements, Float NaN / ±0 / ±inf"""
    cols, row, n_rows = hand_built(oracle_mod)
    rel = pg.relation(95, "public", "pq", "f", sc.rel_cols(cols, set()))
    w = pg.StreamWriter()
    tx = sc.Tx(w)
    tx.begin()
    w.emit(rel)
    for r in range(n_rows):
        w.emit(pg.insert(95, row(r)))
        if r % 3 == 1:
            w.emit(pg.update(95, row(r + 1), old=row(r)))
        if r % 5 == 2:
            w.emit(pg.delete(95, old=row(r)))
    tx.commit()
    assert run_stream(gpu, {95: cols}, w.bytes(), "hand-built", required=(0,)) > 0


def _copy_check(gpu, oids, rows, what, required=(), slices=()):
    lib = abi.load()
    dec = gpu.Decoder(0)
    dec.put_table_schema(7, [dict(name=f"c{i}", type_oid=o, pk=1 if i == 0 else None, nullable=True) for i, o in enumerate(oids)])
    with copy_batch(gpu, dec, 7, rows) as bh:
        a = _emit(lib, bh, 0)
        cols = emit_columns(lib, a)
        n = lib.etl_dec_arrow_rows(a)
        fields = fields_for(cols, required)
        check_write(lib, a, cols, fields, 0, n, what, cdc_ratio=True)
        for rb, re in slices:
            check_write(lib, a, cols, fields, rb, re, f"{what} [{rb}, {re})")
        lib.etl_dec_arrow_free(a)
    dec.close()


def test_copy_batch(gpu):
    oids, rows = synth_rows(30000, 77)
    _copy_check(gpu, oids, rows, "copy", required=(0,), slices=[(19999, 20001), (5, 29000)])


def test_long_text_across_page_cuts(gpu):
    """values of 5 MiB, 300 KiB and a few bytes: pages end after the row that reaches 1 MiB; > 64-byte min / max"""
    rng = np.random.default_rng(5)
    rows = []
    for r in range(25000):
        k = r % 97
        s = "x" * (5 << 20) if r == 12345 else ("y%d" % r) * (30000 if k == 3 else 1)
        if r % 11 == 0:
            s = "\\N"
        rows.append(b"%d\t%s\n" % (int(rng.integers(-2**31, 2**31)), s.encode()))
    _copy_check(gpu, [INT4, TEXT], rows, "long text", slices=[(12345, 12346), (100, 24000)])


def test_lists_across_page_cuts(gpu):
    """List columns past 20 000 rows and 1 MiB of values: int4[] pages cut by bytes, text[] with 40 KiB elements, a
    required bool[] (max definition level 2) whose bit scratch spans pages; NULL arrays, {} and NULL elements"""
    rng = np.random.default_rng(17)
    rows = []
    for r in range(30000):
        k = int(rng.integers(0, 61))
        ints = "\\N" if r % 13 == 0 else "{}" if r % 17 == 0 else "{%s}" % ",".join("NULL" if (r + j) % 11 == 0 else str(r * 7 + j) for j in range(k))
        bools = "{%s}" % ",".join(("t", "f", "NULL")[(r + j) % 3] for j in range(r % 6))
        texts = "\\N" if r % 19 == 0 else "{%s}" % ",".join(("w" * 40960 if r % 500 == 7 else "s%d" % (r + j)) if (r + j) % 5 else "NULL"
                                                             for j in range(r % 4))
        rows.append(("%d\t%s\t%s\t%s\n" % (r, ints, bools, texts)).encode())
    _copy_check(gpu, [INT4, 1007, 1000, 1009], rows, "lists", required=(0, 2), slices=[(19999, 20002), (7, 29000)])


def test_two_row_groups(gpu):
    n = (1 << 20) + 4321
    rows = [b"%d\tv%d\n" % (i * 7 - 5, i % 1000) if i % 17 else b"\\N\t\\N\n" for i in range(n)]
    _copy_check(gpu, [INT4, TEXT], rows, "two row groups", slices=[((1 << 20) - 3, (1 << 20) + 3)])


def test_required_null_and_arguments(gpu, oracle_mod):
    lib = abi.load()
    dec = gpu.Decoder(0)
    oids = [INT4, TEXT]
    dec.put_table_schema(7, [dict(name=f"c{i}", type_oid=o, pk=None, nullable=True) for i, o in enumerate(oids)])
    rows = [b"%d\tt%d\n" % (i, i) if i not in (700, 900) else b"\\N\t\\N\n" for i in range(1000)]
    with copy_batch(gpu, dec, 7, rows) as bh:
        a = _emit(lib, bh, 0)
        cols = emit_columns(lib, a)
        col, row = C.c_uint32(), C.c_uint64()
        for req, rb, want in (((1,), 0, (1, 700)), ((0, 1), 0, (0, 700)), ((0,), 701, (0, 900))):
            rc, h = pq_write(lib, a, fields_for(cols, req), rb, 1000, abi.PQ_SNAPPY)
            assert rc == 0 and lib.etl_dec_parquet_size(h) == 0 and not lib.etl_dec_parquet_bytes(h, 1)
            assert lib.etl_dec_parquet_required_null(h, C.byref(col), C.byref(row)) == 0
            assert (col.value, row.value) == want
            lib.etl_dec_parquet_free(h)
        rc, h = pq_write(lib, a, fields_for(cols), 0, 1000, abi.PQ_SNAPPY)
        assert rc == 0 and lib.etl_dec_parquet_required_null(h, C.byref(col), C.byref(row)) == 0
        assert (col.value, row.value) == (2**32 - 1, 2**64 - 1)
        lib.etl_dec_parquet_free(h)
        good = fields_for(cols)
        bad = [(good[:-1], 0, 1000, 0), (good, 5, 4, 0), (good, 0, 1001, 0), (good, 0, 10, 2),
               ([(b"", 1, 0, 0)] + good[1:], 0, 10, 0), ([(b"x" * 1025, 1, 0, 0)] + good[1:], 0, 10, 0)]
        for f, rb, re, codec in bad:
            assert pq_write(lib, a, f, rb, re, codec)[0] == ERR_INVALID_ARG
        arr = (abi.ParquetField * len(good))()
        for i, g in enumerate(good):
            arr[i].name, arr[i].field_id = g[0].encode(), g[1]
        arr[0].name = None
        h = C.c_void_p()
        assert lib.etl_dec_parquet_write(a, arr, len(good), 0, 10, 0, 1, C.byref(h)) == ERR_INVALID_ARG
        assert pq_write(lib, a, [(b"x" * 1024, 1, 0, 0)] + good[1:], 0, 10, 0)[0] == 0
        lib.etl_dec_arrow_free(a)
        # an emit without ETL_ARROW_ALL_COLUMNS has no unsupported column here; one with a Json column does
    dec.put_table_schema(9, [])                                            # a zero-column table, no CDC columns: no file
    with copy_batch(gpu, dec, 9, [b"\n"] * 3) as bh:
        a = C.c_void_p()
        assert lib.etl_dec_arrow_emit(bh._h, 0, 1 | abi.ARROW_ALL_COLUMNS, 1, C.byref(a)) == 0
        assert lib.etl_dec_arrow_cols(a) == 0
        h = C.c_void_p()
        assert lib.etl_dec_parquet_write(a, None, 0, 0, lib.etl_dec_arrow_rows(a), 0, 1, C.byref(h)) == ERR_INVALID_ARG
        lib.etl_dec_arrow_free(a)
    dec.put_table_schema(8, [dict(name="j", type_oid=3802, pk=None, nullable=True)])
    with copy_batch(gpu, dec, 8, [b'{"a": 1}\n']) as bh:
        a = C.c_void_p()
        assert lib.etl_dec_arrow_emit(bh._h, 0, 1, 1, C.byref(a)) == 0
        assert pq_write(lib, a, [("j", 1, 0, 0)], 0, 1, 0)[0] == ERR_INVALID_ARG
        lib.etl_dec_arrow_free(a)
    dec.close()


def test_write_free_cycles_keep_memory_stable(gpu):
    lib = abi.load()
    dec = gpu.Decoder(0)
    oids, rows = synth_rows(3000, 9)
    dec.put_table_schema(7, [dict(name=f"c{i}", type_oid=o, pk=None, nullable=True) for i, o in enumerate(oids)])
    free, total = C.c_uint64(), C.c_uint64()
    with copy_batch(gpu, dec, 7, rows) as bh:
        a = _emit(lib, bh, 0)
        fields = fields_for(emit_columns(lib, a))
        for i in range(100):
            rc, h = pq_write(lib, a, fields, 0, 3000, i % 2, to_host=i % 3 == 0)
            assert rc == 0 and lib.etl_dec_parquet_size(h) > 0
            lib.etl_dec_parquet_free(h)
            assert lib.etl_dec_mem_info(dec._ctx, C.byref(free), C.byref(total)) == 0
            if i == 1:
                base = free.value
        assert abs(free.value - base) <= 4 << 20, (free.value, base)
        lib.etl_dec_arrow_free(a)
    dec.close()
