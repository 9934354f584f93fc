"""Columnar emitter with ETL_ARROW_ALL_COLUMNS (csrc/arrow_emit.cu, csrc/arrow_format.cuh): Numeric and Json columns as
cell_to_string's Utf8 text and array columns as List<child>, against the Python restatements of the reference's
encoders (tests/arrow_ref.py) evaluated on the ORACLE's planes.  The columns the emitter already built must be
byte-identical to an emit without the bit."""
import ctypes as C

import numpy as np
import pytest

import arrow_ref as R
import scenarios as sc
from etl_b200 import abi, pgoutput as pg, workloads as wl

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def gpu():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from etl_b200 import decoder
    return decoder


def bits(ptr, n):
    raw = np.frombuffer((C.c_uint8 * ((n + 7) // 8)).from_address(ptr), dtype=np.uint8) if n else np.zeros(0, np.uint8)
    return np.unpackbits(raw, bitorder="little")[:n].astype(bool)


def arr(ptr, ctype, dtype, n):
    return np.frombuffer((ctype * n).from_address(ptr), dtype=dtype) if n else np.zeros(0, dtype)


def raw_column(lib, a, c, n):
    """every buffer of a column as bytes / arrays (host image), for byte-identity checks"""
    col = abi.ArrowColumn()
    assert lib.etl_dec_arrow_column(a, c, 1, C.byref(col)) == 0
    out = [col.arrow_type]
    if col.arrow_type and n:
        out.append(bytes((C.c_uint8 * ((n + 7) // 8)).from_address(col.validity)))
        width = {1: None, 2: 4, 3: 8, 4: 4, 5: 8, 8: 4, 9: 8, 10: 8, 11: 8, 12: 16}.get(col.arrow_type)
        if col.arrow_type == 1:
            out.append(bytes((C.c_uint8 * ((n + 7) // 8)).from_address(col.values)))
        elif width:
            out.append(bytes((C.c_uint8 * (n * width)).from_address(col.values)))
        else:
            ow = 4 if col.arrow_type == 6 else 8
            out.append(bytes((C.c_uint8 * ((n + 1) * ow)).from_address(col.offsets)))
            out.append(bytes((C.c_uint8 * col.data_bytes).from_address(col.data)) if col.data_bytes else b"")
    return out


def check_utf8(col, n, want, what):
    _, valid, offs, data = want
    assert col.arrow_type == R.A_UTF8, what
    if not n:
        return
    assert np.array_equal(bits(col.validity, n), valid), f"validity of {what}"
    got_offs = arr(col.offsets, C.c_int32, np.int32, n + 1).astype(np.int64)
    if not np.array_equal(got_offs, offs):
        i = int(np.nonzero(got_offs != offs)[0][0])
        raise AssertionError(f"offsets of {what} differ at {i}: {got_offs[max(0, i - 1):i + 2]} vs {offs[max(0, i - 1):i + 2]}")
    got = bytes((C.c_uint8 * col.data_bytes).from_address(col.data)) if col.data_bytes else b""
    if got != data:
        i = next(k for k in range(n) if got[offs[k]:offs[k + 1]] != data[offs[k]:offs[k + 1]])
        raise AssertionError(f"{what} row {i}: {got[offs[i]:offs[i + 1]][:200]!r} != {data[offs[i]:offs[i + 1]][:200]!r}")


CHILD_NP = {R.A_I32: (C.c_int32, np.int32), R.A_DATE32: (C.c_int32, np.int32), R.A_F32: (C.c_uint32, np.uint32),
            R.A_I64: (C.c_int64, np.int64), R.A_TIME64: (C.c_int64, np.int64), R.A_TS: (C.c_int64, np.int64),
            R.A_TSTZ: (C.c_int64, np.int64), R.A_F64: (C.c_uint64, np.uint64)}


def check_list(lib, a, c, col, n, want, what):
    _, valid, loffs, ct, cvalid, child = want
    assert col.arrow_type == R.A_LIST, what
    assert not col.values and not col.data, what
    kid, ne = abi.ArrowColumn(), C.c_uint64()
    assert lib.etl_dec_arrow_list_child(a, c, 1, C.byref(kid), C.byref(ne)) == 0
    assert kid.arrow_type == ct, (what, kid.arrow_type, ct)
    if not n:
        return
    assert np.array_equal(bits(col.validity, n), valid), f"list validity of {what}"
    assert np.array_equal(arr(col.offsets, C.c_int32, np.int32, n + 1).astype(np.int64), loffs), f"list offsets of {what}"
    ne = ne.value
    assert ne == int(loffs[-1]), what
    if not ne:
        return
    assert np.array_equal(bits(kid.validity, ne), cvalid), f"child validity of {what}"
    if ct == R.A_UTF8:
        check_utf8(kid, ne, ("utf8", cvalid) + child, f"child of {what}")
    elif ct == R.A_LBIN:
        coffs, data = child
        assert np.array_equal(arr(kid.offsets, C.c_int64, np.int64, ne + 1), coffs), what
        assert bytes((C.c_uint8 * len(data)).from_address(kid.data)) == data if data else kid.data_bytes == 0
    elif ct == R.A_BOOL:
        got = bits(kid.values, ne)
        assert all(bool(g) == w for g, w in zip(got, child) if w is not None), what
    elif ct == R.A_UUID:
        got = bytes((C.c_uint8 * (16 * ne)).from_address(kid.values))
        assert all(got[16 * i:16 * i + 16] == w for i, w in enumerate(child) if w is not None), what
    else:
        ctype, dt = CHILD_NP[ct]
        got = arr(kid.values, ctype, dt, ne)
        for i, w in enumerate(child):
            if w is not None:
                assert int(got[i]) == (w & 0xFFFFFFFFFFFFFFFF if dt == np.uint64 else w), (what, i, int(got[i]), w)


def emit(lib, bh, si, kinds):
    a = C.c_void_p()
    rc = lib.etl_dec_arrow_emit(bh._h, si, kinds, 1, C.byref(a))
    assert rc == 0, rc
    return a


def check_batch(lib, bh, planes, raw, si, kinds):
    """one schema version: the formatted columns against the restatement, the others byte-identical to the emit
    without ETL_ARROW_ALL_COLUMNS; returns the number of rows"""
    recs, want = R.expected_formatted_columns(planes, raw, si, kinds)
    plain, full = emit(lib, bh, si, kinds), emit(lib, bh, si, kinds | R.ALL_COLUMNS)
    try:
        n = lib.etl_dec_arrow_rows(full)
        assert n == lib.etl_dec_arrow_rows(plain) == len(recs)
        if n:
            got_recs = arr(lib.etl_dec_arrow_row_records(full, 1), C.c_uint64, np.uint64, n)
            assert np.array_equal(got_recs, np.array(recs, dtype=np.uint64))
        n_cols = lib.etl_dec_arrow_cols(full)
        for c in range(n_cols):
            if c in want:
                assert raw_column(lib, plain, c, n) == [R.A_UNSUP]
                col = abi.ArrowColumn()
                assert lib.etl_dec_arrow_column(full, c, 1, C.byref(col)) == 0
                if want[c][0] == "utf8":
                    check_utf8(col, n, want[c], f"column {c}")
                else:
                    check_list(lib, full, c, col, n, want[c], f"column {c}")
            else:
                assert raw_column(lib, full, c, n) == raw_column(lib, plain, c, n), f"column {c} changed"
        return n, want
    finally:
        lib.etl_dec_arrow_free(plain)
        lib.etl_dec_arrow_free(full)


def decode(gpu, oracle_mod, tables, raw):
    orc = oracle_mod.Oracle()
    dec = gpu.Decoder(0)
    for tid, cols in tables.items():
        orc.put_table_schema(tid, cols)
        dec.put_table_schema(tid, cols)
    st = gpu.Stager(len(raw) + 64, 2048)
    st.append_framed(raw)
    return orc.decode(raw), dec, st


@pytest.mark.parametrize("name,scale,kinds", [("c3", 0.001, 3), ("c3", 0.001, 7), ("c4", 0.002, 3), ("c4", 0.002, 7)])
def test_formatted_columns_match_reference_encoders(gpu, oracle_mod, name, scale, kinds):
    w = wl.make(name, scale, n_segments=1)
    stream, _ = w.generate()
    raw = stream.tobytes()
    planes, dec, st = decode(gpu, oracle_mod, w.table_schemas(), raw)
    lib = abi.load()
    n_formatted = 0
    with dec.decode_input(st.view(), to_host=True) as bh:
        for si in range(len(planes.schemas)):
            n, want = check_batch(lib, bh, planes, raw, si, kinds)
            n_formatted += n * len(want)
    assert n_formatted > 0
    st.close()
    dec.close()


NUMERICS = ["NaN", "Infinity", "-Infinity", "-0.00", "1e100", "1e-100", "0.0012000", "1" + "0" * 60 + "." + "0" * 900 + "1", "-123.450",
            "9999.9999", "10000.0001", "0", "120.00"]
DOCS = ['{"key": "value"}', ' {"b":1, "a":[1 ,2,{"z":null}],"b":2} ', '[1.50, -0, 1E+5, 12345678901234567890123]',
        '"\\u00e9\\ud83d\\ude00\\/\\u0000\\u001f\\b"', '{"k10":1,"k2":2,"\\u00e9":3,"é":4,"z":{"y":1,"y":[{"a":1,"a":2}]}}', "null",
        "{}", "[]", '{"\\u0061":1,"a":2}', " true ", '{"esc":"a\\\\b\\"c\\/d\\r\\n\\t\\f"}']


def _big_doc():
    members = ['"k%d": {"v": [%d, "s%d\\n", {"x%d": null, "x%d": true}], "k%d": %d}' % (i % 5000, i, i, i % 7, i % 7, i % 3, i) for i in range(6000)]
    doc = "{" + ", ".join(members) + "}"
    assert len(doc) >= 256 * 1024
    return doc


def test_hand_built_stream(gpu, oracle_mod):
    """numeric edge cases, the JSON cases and one document >= 256 KiB, every valid array spelling of the parity tests
    plus NULL arrays and {}: in inserts, Full updates and deletes with a Full old image"""
    from test_gpu_parity import ARRAY_COLS
    usable = [(oid, v) for oid, v, _ in ARRAY_COLS if oracle_mod.kind_for_oid(oid) & 0x20]
    cols = [sc.col("id", sc.INT8, 1), sc.col("n", sc.NUMERIC, None, True), sc.col("j", sc.JSONB, None, True),
            sc.col("j2", 114, None, True)] + [sc.col(f"a{oid}", oid, None, True) for oid, _ in usable]
    rel = pg.relation(93, "public", "fmt", "f", sc.rel_cols(cols, set()))
    docs = DOCS + [_big_doc()]

    def row(r):
        arrays = []
        for j, (_, v) in enumerate(usable):
            k = (r + j) % (len(v) + 2)
            arrays.append(None if k == len(v) else ("{}" if k == len(v) + 1 else v[k]))
        doc = docs[r % len(docs)] if r % 9 else None
        return [str(r), NUMERICS[r % len(NUMERICS)] if r % 11 else None, doc, docs[(r * 7) % len(docs)]] + arrays
    w = pg.StreamWriter()
    tx = sc.Tx(w)
    tx.begin()
    w.emit(rel)
    n_rows = 3 * len(docs) * 4
    for r in range(n_rows):
        w.emit(pg.insert(93, row(r)))
        if r % 3 == 1:
            w.emit(pg.update(93, row(r + 1), old=row(r)))
        if r % 5 == 2:
            w.emit(pg.delete(93, old=row(r)))
    tx.commit()
    raw = w.bytes()
    planes, dec, st = decode(gpu, oracle_mod, {93: cols}, raw)
    assert planes.first_error[0] is None, planes.first_error
    lib = abi.load()
    with dec.decode_input(st.view(), to_host=True) as bh:
        for kinds in (1, 2, 4, 7):
            n, want = check_batch(lib, bh, planes, raw, 0, kinds)
            assert n > 0
            assert {c for c, x in want.items() if x[0] == "list"} == set(range(4, len(cols)))
        # a second implementation of serde_json's Display: the shim's tree printer, on the inserts' and updates' new rows
        full = emit(lib, bh, 0, 3 | R.ALL_COLUMNS)
        lst = C.c_void_p()
        assert lib.etl_shim_materialise(bh._h, st.view().host_buf, None, C.byref(lst)) == 0
        recs = arr(lib.etl_dec_arrow_row_records(full, 1), C.c_uint64, np.uint64, lib.etl_dec_arrow_rows(full))
        event_of = np.cumsum((planes.rec_flags[:planes.n_records] & 0x80) != 0) - 1
        buf = C.create_string_buffer(1 << 20)
        n_cross = 0
        for c in (2, 3):
            col = abi.ArrowColumn()
            assert lib.etl_dec_arrow_column(full, c, 1, C.byref(col)) == 0
            offs = arr(col.offsets, C.c_int32, np.int32, len(recs) + 1)
            valid = bits(col.validity, len(recs))
            data = bytes((C.c_uint8 * col.data_bytes).from_address(col.data))
            for i, r in enumerate(recs):
                k = lib.etl_shim_json_text(lst, int(event_of[int(r)]), c, buf, len(buf))
                assert (k >= 0) == bool(valid[i]), (c, i)
                if k >= 0:
                    assert buf.raw[:k] == data[offs[i]:offs[i + 1]], (c, i)
                    n_cross += 1
        assert n_cross > len(recs)
        lib.etl_shim_event_list_free(lst)
        lib.etl_dec_arrow_free(full)
    st.close()
    dec.close()


def test_rows_after_a_data_error_are_not_emitted(gpu, oracle_mod):
    cols = [sc.col("id", sc.INT8, 1), sc.col("n", sc.NUMERIC, None, True), sc.col("j", sc.JSONB, None, True),
            sc.col("a", 1231, None, True)]
    rel = pg.relation(94, "public", "err", "d", sc.rel_cols(cols, {"id"}))
    w = pg.StreamWriter()
    tx = sc.Tx(w)
    tx.begin()
    w.emit(rel)
    for r in range(40):
        w.emit(pg.insert(94, [str(r), "%d.5" % r if r != 23 else "1.2.3", '{"r":%d,"a":[%d]}' % (r, r), "{%d,NULL,1.50}" % r]))
    tx.commit()
    raw = w.bytes()
    planes, dec, st = decode(gpu, oracle_mod, {94: cols}, raw)
    assert planes.first_error[0] is not None
    lib = abi.load()
    with dec.decode_input(st.view(), to_host=True) as bh:
        assert bh.summary().first_error.record_index == planes.first_error[0]
        n, want = check_batch(lib, bh, planes, raw, 0, 7)
        assert n == 23
        assert want[1][3].endswith(b"22.5")
    st.close()
    dec.close()
