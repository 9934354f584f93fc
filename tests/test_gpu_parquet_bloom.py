"""Bloom filters of etl_dec_parquet_write_bloom (csrc/parquet_write.cu) against the Python restatement
(tests/parquet_bloom_ref.py) fed the same Arrow emit's columns.  Every input is written in {UNCOMPRESSED, SNAPPY} ×
{with, without ETL_PQ_DICTIONARY} × {with, without ETL_PQ_PAGE_INDEX}, with filters on every eligible column under two
settings (fpp 0.01 with the chunk's count as ndv; mixed fpp, explicit ndv and a max_bytes cap that bites), and checked:
the file equals with_bloom applied to the same call's file without filters; the bytes before the filters and the page
index structs are unchanged; fields 14 / 15 point at a header whose numBytes plus its length is the stated length;
every non-null value tests positive; the filters are the same with and without the dictionary; the metrics are those of
the file without filters; pyarrow reads the values; a second write gives the same bytes; bloom NULL and all-zero fpp
give the file without filters.  Inputs: c1–c5 (every schema version), a 200 000-row COPY batch, a hand-built table of
every leaf type, an edge table (−0.0 / NaN, empty and long strings, null and empty lists, an all-null column), two row
groups, row slices and zero rows; then required-null files and the argument checks."""
import ctypes as C

import numpy as np
import pytest

import parquet_bloom_ref as B
import parquet_index_ref as X
import parquet_ref as R
import scenarios as sc
from parquet_io import emit_columns, fields_for, file_bytes, metrics, pq_write, pq_write_bloom
from etl_b200 import abi, pgoutput as pg, workloads as wl
from test_gpu_arrow_copy import copy_batch
from test_gpu_copy import synth_rows
from test_gpu_parquet import ERR_INVALID_ARG, INT4, TEXT, _decode_stream, _emit, check_pyarrow
from test_gpu_rowbinary import hand_built

pytestmark = pytest.mark.gpu

PIDX, DICT = abi.PQ_PAGE_INDEX, abi.PQ_DICTIONARY
FLOAT8, BYTEA, BOOL, INT4_ARR, TEXT_ARR = 701, 17, 16, 1007, 1009
CODECS = [c | d | p for c in (abi.PQ_UNCOMPRESSED, abi.PQ_SNAPPY) for d in (0, DICT) for p in (0, PIDX)]


@pytest.fixture(scope="module")
def gpu():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from etl_b200 import decoder
    return decoder


def _write(lib, a, fields, bloom, rb, re, codec):
    rc, h = pq_write_bloom(lib, a, fields, bloom, rb, re, codec)
    assert rc == 0, hex(codec)
    data = file_bytes(lib, h)
    m = metrics(lib, h, len(fields))
    lib.etl_dec_parquet_free(h)
    return data, m


def settings(cols, fields):
    """the two filter settings of the module docstring (Boolean leaves get fpp 0)"""
    leaves = [R.Leaf(c, f) for c, f in zip(cols, fields)]
    ok = [leaf.atype != R.BOOLEAN for leaf in leaves]
    auto = [(0.01, 0, 0) if e else (0.0, 0, 0) for e in ok]
    mixed = [((0.05, 0, 64), (0.1, 1000, 0), (0.001, 50, 1 << 27), (0.3, 0, 1 << 20))[i % 4] if e else (0.0, 0, 0)
             for i, e in enumerate(ok)]
    return [auto, mixed]


def _no_false_negatives(cols, fields, rb, re, got):
    leaves = [R.Leaf(c, f) for c, f in zip(cols, fields)]
    k = 0
    for g0 in range(rb, re, R.ROW_GROUP_ROWS):
        g1 = min(re, g0 + R.ROW_GROUP_ROWS)
        for leaf in leaves:
            if got[k] is not None:
                bits = got[k][4]
                for h in B.chunk_hashes(leaf, *leaf.items(g0, g1))[:2000]:
                    assert B.contains(bits, int(h)), (leaf.name, k)
            k += 1


def check_bloom(lib, a, cols, fields, rb, re, what, codecs=CODECS, pyarrow=True):
    for si, bloom in enumerate(settings(cols, fields)):
        filters = B.chunk_filters(cols, fields, rb, re, bloom)
        seen = {}
        for codec in codecs:
            w = f"{what} setting {si} codec {codec:#x}"
            base, base_m = _write(lib, a, fields, None, rb, re, codec)
            got, got_m = _write(lib, a, fields, bloom, rb, re, codec)
            want = B.with_bloom(base, cols, fields, rb, re, bloom, filters)
            if got != want:
                at = next((i for i in range(min(len(got), len(want))) if got[i] != want[i]), min(len(got), len(want)))
                raise AssertionError(f"{w}: file with filters differs at byte {at} of {len(want)} (got {len(got)})")
            assert got_m == base_m, w
            if rb == re:
                assert got == base, w
                continue
            end = B.data_end(base)
            assert got[:end] == base[:end], w
            if codec & PIDX:
                assert X.read_indexes(got) == X.read_indexes(base), w
            read = B.read_filters(got)
            for f in read:
                if f is not None:
                    off, length, hdr, hb, bits = f
                    assert hdr[1] + len(hb) == length and len(bits) == hdr[1], w
            seen.setdefault(codec & ~DICT, []).append([f and f[4] for f in read])
            if si == 0 and codec == codecs[0]:
                _no_false_negatives(cols, fields, rb, re, read)
                assert _write(lib, a, fields, bloom, rb, re, codec)[0] == got, f"{w}: a second write differs"
                assert _write(lib, a, fields, [(0.0, 0, 0)] * len(fields), rb, re, codec)[0] == base, w
            if pyarrow and codec & 0xFF == abi.PQ_SNAPPY and not codec & DICT:
                check_pyarrow(got, cols, fields, rb, re)
        for k, v in seen.items():                          # with and without the dictionary
            assert all(x == v[0] for x in v), f"{what} setting {si}"


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
            check_bloom(lib, a, cols, fields, 0, n, f"{what} v{si}")
            if n > 2:
                check_bloom(lib, a, cols, fields, n // 3, n - n // 4, f"{what} v{si} slice", codecs=CODECS[::3])
                check_bloom(lib, a, cols, fields, n // 2, n // 2, f"{what} v{si} empty", codecs=CODECS[::5])
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


def _copy_check(gpu, oids, rows, what, required=(), slices=(), codecs=CODECS, pyarrow=True):
    lib = abi.load()
    dec = gpu.Decoder(0)
    dec.put_table_schema(7, [dict(name=f"c{i}", type_oid=o, pk=1 if i == 0 else None, nullable=True) for i, o in enumerate(oids)])
    with copy_batch(gpu, dec, 7, rows) as bh:
        a = _emit(lib, bh, 0)
        cols = emit_columns(lib, a)
        n = lib.etl_dec_arrow_rows(a)
        fields = fields_for(cols, required)
        check_bloom(lib, a, cols, fields, 0, n, what, codecs, pyarrow)
        for rb, re in slices:
            check_bloom(lib, a, cols, fields, rb, re, f"{what} [{rb}, {re})", codecs[::3], pyarrow)
        lib.etl_dec_arrow_free(a)
    dec.close()


def test_copy_batch_200k(gpu):
    oids, rows = synth_rows(200000, 41)
    _copy_check(gpu, oids, rows, "copy 200k", required=(0,), slices=[(19999, 20001), (5, 150000), (7, 7)])


def test_edges(gpu):
    """−0.0 / +0.0 / NaN, empty, short and long (≥ 1 KiB) text and bytea, null and empty lists with null elements, an
    all-null column, a Boolean column (no filter)"""
    n = 30000
    rows = []
    for r in range(n):
        k = r % 7
        text = "\\N" if r % 13 == 0 else "" if k == 0 else "t" if k == 1 else ("é%d" % r) * (300 if k == 2 else 3)
        byt = "\\\\x" + ("" if k == 0 else "%02x" % (r % 256) * (1100 if k == 1 else 5))
        fl = ("NaN", "0", "-0", "-%d.5" % r, "%d.25" % (r % 500))[r % 5]
        ints = "\\N" if r % 17 == 0 else "{}" if r % 19 == 0 else "{%s}" % ",".join("NULL" if (r + j) % 11 == 0 else str(r - j) for j in range(r % 5))
        texts = "{%s}" % ",".join('"%s"' % ("w" * (j * 40) + str(r)) if (r + j) % 3 else "NULL" for j in range(r % 3))
        rows.append(("%d\t%s\t%s\t%s\t\\N\t%s\t%s\t%s\n" % (r, text, byt, fl, "t" if r % 2 else "f", ints, texts)).encode())
    _copy_check(gpu, [INT4, TEXT, BYTEA, FLOAT8, INT4, BOOL, INT4_ARR, TEXT_ARR], rows, "edges", required=(0,),
                slices=[(19990, 20010), (1, 2)])


def test_two_row_groups(gpu):
    n = (1 << 20) + 4321
    rows = [b"%d\tv%d\n" % (i * 7 - 5, i % 1000) if i % 17 else b"\\N\t\\N\n" for i in range(n)]
    _copy_check(gpu, [INT4, TEXT], rows, "two row groups", slices=[((1 << 20) - 3, (1 << 20) + 3)],
                codecs=[abi.PQ_SNAPPY, abi.PQ_SNAPPY | DICT | PIDX], pyarrow=False)


def test_required_null_and_arguments(gpu):
    lib = abi.load()
    dec = gpu.Decoder(0)
    dec.put_table_schema(7, [dict(name="c0", type_oid=INT4, pk=None, nullable=True), dict(name="c1", type_oid=TEXT, pk=None, nullable=True),
                             dict(name="c2", type_oid=BOOL, pk=None, nullable=True)])
    rows = [b"%d\t%s\tt\n" % (i % 4, b"\\N" if i == 500 else b"t%d" % (i % 3)) for i in range(1000)]
    with copy_batch(gpu, dec, 7, rows) as bh:
        a = _emit(lib, bh, 0)
        cols = emit_columns(lib, a)
        fields = fields_for(cols)
        nf = len(fields)
        ok = [(0.01, 0, 0), (0.01, 0, 32), (0.0, 0, 1 << 27)] + [(0.5, 1, 0)] * (nf - 3)
        for codec in CODECS:
            rc, h = pq_write_bloom(lib, a, fields, ok, 0, 1000, codec)
            assert rc == 0 and lib.etl_dec_parquet_size(h) > 0
            lib.etl_dec_parquet_free(h)
        # a null in a required column: no file, with or without filters
        req = fields_for(cols, required=(1,))
        rc, h = pq_write_bloom(lib, a, req, ok, 0, 1000, abi.PQ_SNAPPY)
        col, row = C.c_uint32(), C.c_uint64()
        assert rc == 0 and lib.etl_dec_parquet_size(h) == 0
        assert lib.etl_dec_parquet_required_null(h, C.byref(col), C.byref(row)) == 0 and (col.value, row.value) == (1, 500)
        lib.etl_dec_parquet_free(h)
        bad = [(float("nan"), 0, 0), (-0.1, 0, 0), (1.0, 0, 0), (1.5, 0, 0), (0.01, 0, 48), (0.01, 0, 16), (0.01, 0, 1 << 28),
               (0.01, 0, 3), (0.0, 0, 100)]
        for b in bad:
            arr = [b] + ok[1:]
            assert pq_write_bloom(lib, a, fields, arr, 0, 1000, abi.PQ_SNAPPY)[0] == ERR_INVALID_ARG, b
        boolean = ok[:2] + [(0.01, 0, 0)] + ok[3:]                                  # c2 is Boolean
        assert pq_write_bloom(lib, a, fields, boolean, 0, 1000, abi.PQ_SNAPPY)[0] == ERR_INVALID_ARG
        assert pq_write_bloom(lib, a, fields, ok, 0, 1000, abi.PQ_SNAPPY | 0x200)[0] == ERR_INVALID_ARG
        # bloom NULL is etl_dec_parquet_write's file
        for codec in CODECS:
            rc, h = pq_write(lib, a, fields, 0, 1000, codec)
            old = file_bytes(lib, h)
            lib.etl_dec_parquet_free(h)
            assert _write(lib, a, fields, None, 0, 1000, codec)[0] == old
        lib.etl_dec_arrow_free(a)
    dec.close()
