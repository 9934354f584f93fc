"""Parquet writer with ETL_PQ_PAGE_INDEX (csrc/parquet_write.cu) against the Python restatement
(tests/parquet_index_ref.py) fed the same Arrow emit's columns.  Every input is written as {UNCOMPRESSED, SNAPPY} ×
{with, without ETL_PQ_DICTIONARY}, each with and without the flag, and checked: the bytes before the index equal the
file without the flag; the whole file equals the restatement's index added to that file (for Snappy files computed from
that file's own page walk); footer fields 4–7 point at structs of exactly the stated length; PageLocations restart
their first_row_index at each row group; pyarrow reads the values and sees an OffsetIndex on every chunk and a
ColumnIndex exactly where expected; a second write gives the same bytes.  Inputs: c1–c5, a 200 000-row COPY batch, a
hand-built table of truncation, NaN, null and List edges, two row groups, row slices and zero rows; then
sequence_number's boundary order on a c5 emit and the flag's argument checks."""
import ctypes as C

import numpy as np
import pytest

import parquet_index_ref as X
import scenarios as sc
from parquet_io import emit_columns, fields_for, file_bytes, pq_write
from etl_b200 import abi, pgoutput as pg, workloads as wl
from test_gpu_arrow_copy import copy_batch
from test_gpu_copy import synth_rows
from test_gpu_parquet import ERR_INVALID_ARG, INT4, TEXT, _decode_stream, _emit, check_pyarrow
from test_gpu_rowbinary import hand_built

pytestmark = pytest.mark.gpu

PIDX, DICT = abi.PQ_PAGE_INDEX, abi.PQ_DICTIONARY
FLOAT8, BYTEA, INT4_ARR, TEXT_ARR = 701, 17, 1007, 1009
CODECS = [abi.PQ_UNCOMPRESSED, abi.PQ_SNAPPY, abi.PQ_UNCOMPRESSED | DICT, abi.PQ_SNAPPY | DICT]


@pytest.fixture(scope="module")
def gpu():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from etl_b200 import decoder
    return decoder


def _write(lib, a, fields, rb, re, codec):
    rc, h = pq_write(lib, a, fields, rb, re, codec)
    assert rc == 0, hex(codec)
    data = file_bytes(lib, h)
    lib.etl_dec_parquet_free(h)
    return data


def check_index(lib, a, cols, fields, rb, re, what, pyarrow=True):
    """the checks of the module docstring for every codec; returns the parsed indexes of the Snappy dictionary file"""
    import io
    import pyarrow.parquet as pq
    idx = None
    for codec in CODECS:
        w = f"{what} codec {codec:#x}"
        base = _write(lib, a, fields, rb, re, codec)
        got = _write(lib, a, fields, rb, re, codec | PIDX)
        _, foot_at, _ = X.file_footer(base)
        assert got[:foot_at] == base[:foot_at], w
        want = X.with_index(base, cols, fields, rb, re)
        if got != want:
            at = next((i for i in range(min(len(got), len(want))) if got[i] != want[i]), min(len(got), len(want)))
            raise AssertionError(f"{w}: file with the page index differs at byte {at} of {len(want)} (got {len(got)})")
        assert _write(lib, a, fields, rb, re, codec | PIDX) == got, f"{w}: a second write differs"
        if rb == re:
            assert got == base, w
            continue
        fm, _, _ = X.file_footer(got)
        idx = X.read_indexes(got)                         # parses each struct at its stated offset and length
        expect = [ci is not None for ci, _ in X.chunk_indexes(base, cols, fields, rb, re)]
        assert [ci is not None for ci, _ in idx] == expect, w
        k = 0
        for rg in fm[4]:
            for cc in rg[1]:
                locs = idx[k][1][1]
                assert locs[0][3] == 0 and locs[0][1] == cc[3][9], w            # restarts per row group; data_page_offset
                assert all(x[3] < y[3] for x, y in zip(locs, locs[1:])), w
                k += 1
        if pyarrow and codec & 0xFF == abi.PQ_SNAPPY:
            check_pyarrow(got, cols, fields, rb, re)
            md = pq.ParquetFile(io.BytesIO(got)).metadata
            flags = [(md.row_group(g).column(c).has_offset_index, md.row_group(g).column(c).has_column_index)
                     for g in range(md.num_row_groups) for c in range(md.num_columns)]
            assert flags == [(True, e) for e in expect], w
    return idx


def run_stream(gpu, tables, raw, what, required=()):
    lib = abi.load()
    dec, st = _decode_stream(gpu, tables, raw)
    n_total = 0
    with dec.decode_input(st.view(), to_host=True) as bh:
        for si in range(len(bh.schemas())):
            a = _emit(lib, bh, si)
            cols = emit_columns(lib, a)
            n = lib.etl_dec_arrow_rows(a)
            fields = fields_for(cols, required)
            check_index(lib, a, cols, fields, 0, n, f"{what} v{si}")
            if n > 2:
                check_index(lib, a, cols, fields, n // 3, n - n // 4, f"{what} v{si} slice")
                check_index(lib, a, cols, fields, n // 2, n // 2, f"{what} v{si} empty")
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
    tx.commit()
    assert run_stream(gpu, {95: cols}, w.bytes(), "hand-built", required=(0,)) > 0


def _copy_check(gpu, oids, rows, what, required=(), slices=(), pyarrow=True):
    lib = abi.load()
    dec = gpu.Decoder(0)
    dec.put_table_schema(7, [dict(name=f"c{i}", type_oid=o, pk=1 if i == 0 else None, nullable=True) for i, o in enumerate(oids)])
    with copy_batch(gpu, dec, 7, rows) as bh:
        a = _emit(lib, bh, 0)
        cols = emit_columns(lib, a)
        n = lib.etl_dec_arrow_rows(a)
        fields = fields_for(cols, required)
        idx = check_index(lib, a, cols, fields, 0, n, what, pyarrow)
        for rb, re in slices:
            check_index(lib, a, cols, fields, rb, re, f"{what} [{rb}, {re})", pyarrow)
        lib.etl_dec_arrow_free(a)
    dec.close()
    return idx


def test_copy_batch_200k(gpu):
    oids, rows = synth_rows(200000, 41)
    _copy_check(gpu, oids, rows, "copy 200k", required=(0,), slices=[(19999, 20001), (5, 150000)])


def _edge_text(r):
    """Utf8 values of 63, 64, 65 and 200 bytes with 2-, 3- and 4-byte characters across byte 64, and values whose
    character at the cut cannot be incremented"""
    k = r % 12
    if k == 0:
        return "a" * 63
    if k == 1:
        return "b" * 64
    if k == 2:
        return "c" * 65
    if k == 3:
        return "d" * 63 + "é" + "x" * 136                  # 2 bytes at 63..64
    if k == 4:
        return "e" * 62 + "€" + "x" * 135                  # 3 bytes at 62..64
    if k == 5:
        return "f" * 61 + "😀" + "x" * 135                 # 4 bytes at 61..64
    if k == 6:
        return "g" * 60 + "\U0010ffff" + "tail"            # ends at 64: the 'g' before it is incremented
    if k == 7:
        return "h" * 61 + "\uffff" + "tail"
    if k == 8:
        return "i" * 61 + "\ud7ff" + "tail"
    if k == 9:
        return "\U0010ffff" * 20                            # nothing to increment: the whole value
    if k == 10:
        return "\u00e9" * 40
    return "z%d" % r


def test_hand_built_edges(gpu):
    """truncation, bytea, ±0 / NaN-only pages, an all-null and a required column, List columns past 20 000 rows"""
    n = 45000
    rows = []
    for r in range(n):
        k = r % 7
        text = _edge_text(r) if r % 13 else "\\N"
        byt = "\\\\x" + ("ff" * 80 if k == 0 else "00" + "ff" * 70 if k == 1 else "%02x" % (r % 256) * 66 if k == 2 else
                         "ab" * 30 + "ff" * 10 if k == 3 else "%04x" % r)
        fl = "NaN" if r < 20000 else ("0" if k == 0 else "-0" if k == 1 else "%d.5" % (r % 1000 - 500))
        fl2 = ("-0" if r % 2 else "0") if r % 3 else "\\N"
        ints = "\\N" if r % 17 == 0 else "{}" if r % 19 == 0 else "{%s}" % ",".join("NULL" if (r + j) % 11 == 0 else str(r - j) for j in range(r % 5))
        texts = "{%s}" % ",".join('"%s"' % ("w" * 70 + str(j)) if (r + j) % 3 else "NULL" for j in range(r % 3))
        rows.append(("%d\t%s\t%s\t%s\t%s\t\\N\t%s\t%s\n" % (r, text, byt, fl, fl2, ints, texts)).encode())
    idx = _copy_check(gpu, [INT4, TEXT, BYTEA, FLOAT8, FLOAT8, INT4, INT4_ARR, TEXT_ARR], rows, "edges", required=(0,),
                      slices=[(19990, 20010), (20000, 45000), (1, 2)])
    assert idx[3][0] is None and idx[4][0] is not None    # the NaN-only first page: no ColumnIndex
    assert idx[0][0][4] == X.ASCENDING and idx[5][0][1] == [True, True, True]   # the all-null column


def test_two_row_groups(gpu):
    n = (1 << 20) + 4321
    rows = [b"%d\tv%d\n" % (i * 7 - 5, i % 1000) if i % 17 else b"\\N\t\\N\n" for i in range(n)]
    idx = _copy_check(gpu, [INT4, TEXT], rows, "two row groups", slices=[((1 << 20) - 3, (1 << 20) + 3)], pyarrow=False)
    assert len(idx) == 2 * 4


def test_sequence_number_ascending(gpu):
    """a c5 emit of more than 20 000 rows: sequence_number's pages ascend, so readers can binary-search them"""
    lib = abi.load()
    w = wl.make("c5", 0.02, n_segments=1)
    stream, _ = w.generate()
    dec, st = _decode_stream(gpu, w.table_schemas(), stream.tobytes())
    best = 0
    with dec.decode_input(st.view(), to_host=True) as bh:
        for si in range(len(bh.schemas())):
            a = _emit(lib, bh, si)
            cols = emit_columns(lib, a)
            n = lib.etl_dec_arrow_rows(a)
            fields = fields_for(cols)
            if n > 20000:
                best = max(best, n)
                for codec in (abi.PQ_SNAPPY | PIDX, abi.PQ_SNAPPY | DICT | PIDX):
                    data = _write(lib, a, fields, 0, n, codec)
                    ci, oi = X.read_indexes(data)[len(fields) - 1]
                    assert len(oi[1]) > 1 and ci[4] == X.ASCENDING, codec
            lib.etl_dec_arrow_free(a)
    st.close()
    dec.close()
    assert best > 20000


def test_flag_arguments(gpu):
    lib = abi.load()
    dec = gpu.Decoder(0)
    dec.put_table_schema(7, [dict(name="c0", type_oid=INT4, pk=None, nullable=True), dict(name="c1", type_oid=TEXT, pk=None, nullable=True)])
    with copy_batch(gpu, dec, 7, [b"%d\tt%d\n" % (i % 4, i % 3) for i in range(1000)]) as bh:
        a = _emit(lib, bh, 0)
        fields = fields_for(emit_columns(lib, a))
        for codec in CODECS:
            rc, h = pq_write(lib, a, fields, 0, 1000, codec | PIDX)
            assert rc == 0 and lib.etl_dec_parquet_size(h) > 0
            lib.etl_dec_parquet_free(h)
        for codec in (PIDX | 2, 0x800, 0x200 | PIDX, PIDX | DICT | 2):
            assert pq_write(lib, a, fields, 0, 1000, codec)[0] == ERR_INVALID_ARG, hex(codec)
        lib.etl_dec_arrow_free(a)
    dec.close()
