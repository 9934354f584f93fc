"""Parquet writer with ETL_PQ_DICTIONARY (csrc/parquet_write.cu) against the Python restatement (tests/parquet_dict_ref.py,
dictionary=True) fed the same Arrow emit's columns, checked as tests/test_gpu_parquet.py checks the PLAIN file: the
uncompressed file byte for byte, the Snappy file page by page (dictionary pages included), the metrics, and pyarrow's
reading.  Inputs: c1–c5, a COPY batch, every column type with float corners, List columns past 20 000 rows and 1 MiB,
long text across page cuts, two row groups of which one falls back, row slices and zero rows, a low-cardinality COPY
table; then the determinism of the inserts, a file with no eligible chunk, and the flag's argument checks."""
import ctypes as C

import numpy as np
import pytest

import parquet_dict_ref as R
import scenarios as sc
from parquet_io import emit_columns, fields_for, file_bytes, metrics, pq_write
from etl_b200 import abi, pgoutput as pg, workloads as wl
from test_gpu_arrow_copy import copy_batch
from test_gpu_copy import synth_rows
from test_gpu_parquet import EMIT_KINDS, ERR_INVALID_ARG, INT4, TEXT, _decode_stream, _emit, check_pyarrow
from test_gpu_rowbinary import hand_built

pytestmark = pytest.mark.gpu

DICT = abi.PQ_DICTIONARY
BOOL, INT8, DATE, UUID, TEXT_ARR = 16, 20, 1082, 2950, 1009


@pytest.fixture(scope="module")
def gpu():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from etl_b200 import decoder
    return decoder


MASK_CMD = {6, 7, 9, 11}      # ColumnMetaData sizes, data_page_offset, dictionary_page_offset
MASK_RG = {2, 5, 6}


def _masked_footer(fm):
    fm = dict(fm)
    rgs = []
    for rg in fm.get(4, []):
        rg = {k: v for k, v in rg.items() if k not in MASK_RG}
        rg[1] = [{2: None, 3: {k: v for k, v in cc[3].items() if k not in MASK_CMD | {4}}} for cc in rg[1]]
        rgs.append(rg)
    fm[4] = rgs
    return fm


def check_write(lib, a, cols, fields, rb, re, what):
    """the dictionary file, uncompressed and Snappy, against the restatement; returns the uncompressed file"""
    want, want_m, want_pages = R.write(cols, fields, rb, re, dictionary=True)
    rc, h = pq_write(lib, a, fields, rb, re, abi.PQ_UNCOMPRESSED | DICT)
    assert rc == 0, what
    got = file_bytes(lib, h)
    if got != want:
        at = next((i for i in range(min(len(got), len(want))) if got[i] != want[i]), min(len(got), len(want)))
        raise AssertionError(f"{what}: uncompressed dictionary file differs at byte {at} of {len(want)} (got {len(got)})")
    assert metrics(lib, h, len(fields)) == want_m, what
    lib.etl_dec_parquet_free(h)
    import pyarrow as pa
    snappy = pa.Codec("snappy")
    rc, h = pq_write(lib, a, fields, rb, re, abi.PQ_SNAPPY | DICT)
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
        usize[ci] = usize.get(ci, 0) + len(hb) + len(wpayload)
    fm, _ = R.file_footer(data)
    wfm, _ = R.file_footer(want)
    assert _masked_footer(fm) == _masked_footer(wfm), what
    for rg in fm.get(4, []):
        for cc in rg[1]:
            md = cc[3]
            assert md[4] == 1 and cc[2] == md.get(11, md[9]) and (11 not in md or md[11] < md[9])
    got_m = metrics(lib, h, len(fields))
    sizes = ("compressed_bytes", "uncompressed_bytes")
    for g, w in zip(got_m, want_m):
        assert {k: v for k, v in g.items() if k not in sizes} == {k: v for k, v in w.items() if k not in sizes}, what
    for key, per_chunk in zip(sizes, (csize, usize)):
        assert [m[key] for m in got_m] == [sum(per_chunk.get(ci, 0) for ci in range(l, len(per_chunk), len(fields)))
                                           for l in range(len(fields))], (what, key)
    check_pyarrow(data, cols, fields, rb, re)
    lib.etl_dec_parquet_free(h)
    return got


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
            check_write(lib, a, cols, fields, 0, n, f"{what} v{si}")
            if n > 2:
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


def _copy_check(gpu, oids, rows, what, required=(), slices=(), kinds=EMIT_KINDS):
    """the dictionary checks over a COPY batch; returns (uncompressed dictionary file, PLAIN file, decisions per chunk)"""
    lib = abi.load()
    dec = gpu.Decoder(0)
    dec.put_table_schema(7, [dict(name=f"c{i}", type_oid=o, pk=1 if i == 0 else None, nullable=True) for i, o in enumerate(oids)])
    with copy_batch(gpu, dec, 7, rows) as bh:
        a = C.c_void_p()
        assert lib.etl_dec_arrow_emit(bh._h, 0, kinds, 1, C.byref(a)) == 0
        cols = emit_columns(lib, a)
        n = lib.etl_dec_arrow_rows(a)
        fields = fields_for(cols, required) if kinds & abi.ARROW_CDC_COLUMNS else [(f"c{i}", i + 1, 1000 + i, 0) for i in range(len(cols))]
        got = check_write(lib, a, cols, fields, 0, n, what)
        for rb, re in slices:
            check_write(lib, a, cols, fields, rb, re, f"{what} [{rb}, {re})")
        rc, h = pq_write(lib, a, fields, 0, n, abi.PQ_UNCOMPRESSED)
        assert rc == 0
        plain = file_bytes(lib, h)
        lib.etl_dec_parquet_free(h)
        rc, h = pq_write(lib, a, fields, 0, n, abi.PQ_UNCOMPRESSED | DICT)
        assert rc == 0 and file_bytes(lib, h) == got, f"{what}: a second write differs"
        lib.etl_dec_parquet_free(h)
        lib.etl_dec_arrow_free(a)
    dec.close()
    fm, _ = R.file_footer(got)
    return got, plain, [[11 in cc[3] for cc in rg[1]] for rg in fm.get(4, [])]


def test_copy_batch(gpu):
    oids, rows = synth_rows(30000, 77)
    _copy_check(gpu, oids, rows, "copy", required=(0,), slices=[(19999, 20001), (5, 29000)])


def test_long_text_across_page_cuts(gpu):
    rng = np.random.default_rng(5)
    rows = []
    for r in range(25000):
        k = r % 97
        s = "x" * (5 << 20) if r == 12345 else ("y%d" % (r % 5)) * 30000 if k == 3 else "y%d" % (r % 50)
        if r % 11 == 0:
            s = "\\N"
        rows.append(b"%d\t%s\n" % (int(rng.integers(-2**31, 2**31)), s.encode()))
    _, _, dec = _copy_check(gpu, [INT4, TEXT], rows, "long text", slices=[(12345, 12346), (100, 24000), (13000, 24000)])
    assert dec[0][:2] == [True, False]                   # the 5 MiB value passes the limit; without it (13000..) it fits


def test_lists_across_page_cuts(gpu):
    rng = np.random.default_rng(17)
    rows = []
    for r in range(30000):
        k = int(rng.integers(0, 61))
        ints = "\\N" if r % 13 == 0 else "{}" if r % 17 == 0 else "{%s}" % ",".join("NULL" if (r + j) % 11 == 0 else str((r * 7 + j) % 300) for j in range(k))
        bools = "{%s}" % ",".join(("t", "f", "NULL")[(r + j) % 3] for j in range(r % 6))
        texts = "\\N" if r % 19 == 0 else "{%s}" % ",".join(("w" * 40960 if r % 500 == 7 else "s%d" % ((r + j) % 40)) if (r + j) % 5 else "NULL"
                                                             for j in range(r % 4))
        rows.append(("%d\t%s\t%s\t%s\n" % (r, ints, bools, texts)).encode())
    _copy_check(gpu, [INT4, 1007, 1000, TEXT_ARR], rows, "lists", required=(0, 2), slices=[(19999, 20002), (7, 29000)])


def test_two_row_groups_one_falls_back(gpu):
    n = (1 << 20) + 4321
    rows = [b"%d\tv%d\n" % (i * 7 - 5, i % 1000) if i % 17 else b"\\N\t\\N\n" for i in range(n)]
    _, _, dec = _copy_check(gpu, [INT4, TEXT], rows, "two row groups", slices=[((1 << 20) - 3, (1 << 20) + 3)])
    assert dec[0][:2] == [False, True] and dec[1][:2] == [True, True]   # 2^20 distinct ints pass 1 MiB; 4 321 do not


def test_low_cardinality_table(gpu):
    rng = np.random.default_rng(23)
    words = ["active", "pending", "shipped", "cancelled", "returned", "on hold", "lost", "refunded", "draft", "open",
             "closed", "archived"]
    uuids = ["%08x-0000-4000-8000-%012x" % (k * 7919, k) for k in range(9)]
    rows = []
    for r in range(60000):
        tags = "{%s}" % ",".join(("red", "green", "blue", "NULL")[int(x)] for x in rng.integers(0, 4, int(rng.integers(0, 6))))
        rows.append(("%d\t%s\t%d\t2024-03-%02d\t%s\t%s\n" % (
            r, words[int(rng.integers(0, 12))] if r % 23 else "\\N", int(rng.integers(0, 7)), int(rng.integers(1, 29)),
            uuids[int(rng.integers(0, 9))], tags if r % 31 else "\\N")).encode())
    got, plain, dec = _copy_check(gpu, [INT4, TEXT, INT4, DATE, UUID, TEXT_ARR], rows, "low cardinality", required=(0,),
                                  slices=[(100, 50000)])
    assert dec[0][:6] == [True] * 6
    sizes = [[cc[3][7] for cc in R.file_footer(f)[0][4][0][1]] for f in (got, plain)]
    assert all(d * 2 < p for d, p in zip(sizes[0][1:6], sizes[1][1:6])), sizes


def test_duplicates_across_ctas_are_deterministic(gpu):
    """600 000 rows of three values per column: every CTA of the insert pass races on the same slots"""
    rows = [b"%d\t%s\t%d\n" % (i % 3, (b"aa", b"b" * 40, b"c" * 33)[(i * 7) % 3], (i // 5) % 3) for i in range(600000)]
    got, _, dec = _copy_check(gpu, [INT4, TEXT, INT8], rows, "duplicates")
    assert all(dec[0][:3])


def test_no_eligible_chunk_is_the_plain_file(gpu):
    """Boolean columns and columns past the 1 MiB dictionary limit only: the file without the flag, byte for byte"""
    n = 300000
    rows = [b"%s\t%d\t%d\tu%07d\n" % (b"tf"[i % 2:i % 2 + 1] if i % 7 else b"\\N", i * 3 - 1, i * 1000003, i) for i in range(n)]
    got, plain, dec = _copy_check(gpu, [BOOL, INT4, INT8, TEXT], rows, "no dictionary", kinds=7 | abi.ARROW_ALL_COLUMNS)
    assert dec == [[False] * 4] and got == plain


def test_flag_arguments(gpu):
    lib = abi.load()
    dec = gpu.Decoder(0)
    dec.put_table_schema(7, [dict(name="c0", type_oid=INT4, pk=None, nullable=True), dict(name="c1", type_oid=TEXT, pk=None, nullable=True)])
    with copy_batch(gpu, dec, 7, [b"%d\tt%d\n" % (i % 4, i % 3) for i in range(1000)]) as bh:
        a = _emit(lib, bh, 0)
        fields = fields_for(emit_columns(lib, a))
        for codec in (DICT, DICT | abi.PQ_SNAPPY):
            rc, h = pq_write(lib, a, fields, 0, 1000, codec)
            assert rc == 0 and lib.etl_dec_parquet_size(h) > 0
            lib.etl_dec_parquet_free(h)
        for codec in (0x200, 2, DICT | 2, 0x200 | DICT | 1, 0x80000000):
            assert pq_write(lib, a, fields, 0, 1000, codec)[0] == ERR_INVALID_ARG, hex(codec)
        lib.etl_dec_arrow_free(a)
    dec.close()
