"""Columnar emitter on COPY-row batches and the Iceberg CDC columns (csrc/arrow_emit.cu).

* COPY batches (etl_dec_copy_decode → etl_dec_arrow_emit): every column against the tests/arrow_ref.py restatements of
  the reference's encoders, through the per-row entry point of tests/arrow_copy_ref.py, applied to the ORACLE's per-row
  COPY parse (pyoracle.parse_copy_row), with and without ETL_ARROW_ALL_COLUMNS, including text fields that needed
  unescaping (their cells live in the heap, bit 63 of val).
* ETL_ARROW_CDC_COLUMNS on streaming batches: cdc_operation / sequence_number against the restatement on the oracle's
  record planes; every user column byte-identical to an emit without the bit.
* etl_dec_arrow_first_skipped against the oracle's planes."""
import ctypes as C

import numpy as np
import pytest

import arrow_copy_ref as R
import arrow_ref as A
from canon import decode_cell
from etl_b200 import abi, workloads as wl
from test_gpu_arrow_formatted import arr, bits, check_list, check_utf8, raw_column
from test_gpu_copy import JSONB, REF_ROWS, TEXT, INT4, cols_of, synth_rows

pytestmark = pytest.mark.gpu

ALL, CDC = A.ALL_COLUMNS, R.CDC_COLUMNS
NONE = 2**64 - 1
ERR_INVALID_ARG = 1
FIXED_NP = {A.A_I32: (C.c_int32, np.int32), A.A_DATE32: (C.c_int32, np.int32), A.A_F32: (C.c_uint32, np.uint32),
            A.A_I64: (C.c_int64, np.int64), A.A_TIME64: (C.c_int64, np.int64), A.A_TS: (C.c_int64, np.int64),
            A.A_TSTZ: (C.c_int64, np.int64), A.A_F64: (C.c_uint64, np.uint64)}


@pytest.fixture(scope="module")
def gpu():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from etl_b200 import decoder
    return decoder


def copy_batch(gpu, dec, table_id, rows):
    """etl_dec_copy_decode of COPY-text rows (each with its LF), the batch kept open"""
    lib = abi.load()
    offs = np.zeros(len(rows) + 1, dtype=np.uint64)
    offs[1:] = np.cumsum([len(r) for r in rows])
    blob = b"".join(rows)
    padded = np.zeros(len(blob) + 64, dtype=np.uint8)
    padded[:len(blob)] = np.frombuffer(blob, dtype=np.uint8)
    inp = abi.CopyInput()
    inp.host_buf, inp.len, inp.row_offsets, inp.n_rows = padded.ctypes.data, len(blob), offs.ctypes.data, len(rows)
    h = C.c_void_p()
    rc = lib.etl_dec_copy_decode(dec._ctx, table_id, C.byref(inp), abi.RESULTS_TO_HOST, C.byref(h))
    assert rc == 0, lib.etl_dec_last_error(dec._ctx)
    return gpu.BatchHandle(dec, h)


def emit(lib, bh, kinds, si=0):
    a = C.c_void_p()
    rc = lib.etl_dec_arrow_emit(bh._h, si, kinds, 1, C.byref(a))
    assert rc == 0, rc
    return a


def oracle_rows(oracle_mod, oids, rows):
    """the oracle's per-row parse: decoded values of the rows before the first failing one"""
    out = []
    for row in rows:
        e, _, cells, text, heap = oracle_mod.parse_copy_row(oids, row)
        if e:
            break
        out.append([decode_cell(t, v, a, text, heap) for t, v, a in cells])
    return out


def check_column(lib, a, c, n, want, what):
    col = abi.ArrowColumn()
    assert lib.etl_dec_arrow_column(a, c, 1, C.byref(col)) == 0
    form = want[0]
    if form == "unsupported":
        assert col.arrow_type == A.A_UNSUP, what
    elif form == "utf8":
        check_utf8(col, n, want, what)
    elif form == "list":
        check_list(lib, a, c, col, n, want, what)
    elif form == "lbin":
        _, valid, offs, data = want
        assert col.arrow_type == A.A_LBIN, what
        if n:
            assert np.array_equal(bits(col.validity, n), valid), what
            assert np.array_equal(arr(col.offsets, C.c_int64, np.int64, n + 1), offs), what
            assert col.data_bytes == len(data) and (not data or bytes((C.c_uint8 * len(data)).from_address(col.data)) == data), what
    else:
        _, at, valid, values = want
        assert col.arrow_type == at, (what, col.arrow_type, at)
        if not n:
            return
        assert np.array_equal(bits(col.validity, n), valid), f"validity of {what}"
        if at == A.A_BOOL:
            assert [bool(x) for x in bits(col.values, n)] == [bool(v) for v in values], what
        elif at == A.A_UUID:
            assert bytes((C.c_uint8 * (16 * n)).from_address(col.values)) == b"".join(v or b"\0" * 16 for v in values), what
        else:
            ctype, dt = FIXED_NP[at]
            got = arr(col.values, ctype, dt, n)
            want_v = np.array([0 if v is None else (v & NONE if dt == np.uint64 else v) for v in values], dtype=dt)
            assert np.array_equal(got, want_v), what


def check_cdc(lib, a, first, n, p, recs, what):
    """columns first, first + 1: cdc_operation and sequence_number, never null"""
    for c, want in zip((first, first + 1), R.expected_cdc_columns(p, recs)):
        col = abi.ArrowColumn()
        assert lib.etl_dec_arrow_column(a, c, 1, C.byref(col)) == 0
        check_utf8(col, n, want, f"{what}: CDC column {c}")
        if n:
            assert bits(col.validity, n).all()


def check_copy_emit(lib, bh, kinds, want_rows, what):
    """one COPY batch: emits 1 and 1|ALL|CDC (and a mask without bit 0) against the restatement; the columns both
    build are byte-identical.  Returns the number of rows"""
    n_want = len(want_rows)
    plain, full = emit(lib, bh, 1), emit(lib, bh, 1 | ALL | CDC)
    try:
        n = lib.etl_dec_arrow_rows(full)
        assert n == lib.etl_dec_arrow_rows(plain) == n_want, (what, n, n_want)
        assert lib.etl_dec_arrow_cols(plain) == len(kinds) and lib.etl_dec_arrow_cols(full) == len(kinds) + 2
        assert lib.etl_dec_arrow_first_skipped(full) == NONE and lib.etl_dec_arrow_first_skipped(plain) == NONE
        if n:
            assert np.array_equal(arr(lib.etl_dec_arrow_row_records(full, 1), C.c_uint64, np.uint64, n), np.arange(n, dtype=np.uint64))
        want_plain = R.expected_row_columns(kinds, want_rows, False)
        want_full = R.expected_row_columns(kinds, want_rows, True)
        for c in range(len(kinds)):
            check_column(lib, plain, c, n, want_plain[c], f"{what}: column {c}")
            check_column(lib, full, c, n, want_full[c], f"{what}: column {c} (ALL)")
            if want_plain[c][0] != "unsupported":
                assert raw_column(lib, full, c, n) == raw_column(lib, plain, c, n), f"{what}: column {c} changed"
        check_cdc(lib, full, len(kinds), n, None, range(n), what)
    finally:
        lib.etl_dec_arrow_free(plain)
        lib.etl_dec_arrow_free(full)
    none = emit(lib, bh, 6 | ALL | CDC)                    # no inserts selected: no rows, the columns still typed
    try:
        assert lib.etl_dec_arrow_rows(none) == 0 and lib.etl_dec_arrow_cols(none) == len(kinds) + 2
        want_none = R.expected_row_columns(kinds, [], True)
        for c in range(len(kinds)):
            check_column(lib, none, c, 0, want_none[c], f"{what}: column {c} without bit 0")
        check_cdc(lib, none, len(kinds), 0, None, [], what)
    finally:
        lib.etl_dec_arrow_free(none)
    return n


def kinds_of(oracle_mod, oids):
    return [oracle_mod.kind_for_oid(o) for o in oids]


# ------------------------------------------------------------------------------------------------ COPY batches
@pytest.mark.parametrize("idx", range(len(REF_ROWS)))
def test_reference_vectors(gpu, oracle_mod, idx):
    """table_row.rs:206-533, each as a one-row batch; an erroring vector gives zero rows"""
    oids, row = REF_ROWS[idx]
    lib = abi.load()
    dec = gpu.Decoder(0)
    dec.put_table_schema(7, cols_of(oids))
    with copy_batch(gpu, dec, 7, [row]) as bh:
        want = oracle_rows(oracle_mod, oids, [row])
        a = emit(lib, bh, 1 | ALL | CDC)
        try:
            n = lib.etl_dec_arrow_rows(a)
            assert n == len(want)
            assert lib.etl_dec_arrow_cols(a) == len(oids) + 2
            exp = R.expected_row_columns(kinds_of(oracle_mod, oids), want, True)
            for c in range(len(oids)):
                check_column(lib, a, c, n, exp[c], f"vector {idx} column {c}")
            check_cdc(lib, a, len(oids), n, None, range(n), f"vector {idx}")
        finally:
            lib.etl_dec_arrow_free(a)
    dec.close()


@pytest.mark.parametrize("n,bad_at", [(5000, 3777), (200000, None)])
def test_synthetic_tables(gpu, oracle_mod, n, bad_at):
    oids, rows = synth_rows(n, 1234 + n, bad_at)
    lib = abi.load()
    dec = gpu.Decoder(0)
    dec.put_table_schema(7, cols_of(oids))
    with copy_batch(gpu, dec, 7, rows) as bh:
        s = bh.summary()
        assert (s.first_error.record_index == NONE) == (bad_at is None)
        want = oracle_rows(oracle_mod, oids, rows)
        assert len(want) == (n if bad_at is None else bad_at)
        got = check_copy_emit(lib, bh, kinds_of(oracle_mod, oids), want, f"synth {n}")
        assert got == len(want)
    dec.close()


def copy_escape(s: str) -> bytes:
    return s.replace("\\", "\\\\").replace("\t", "\\t").replace("\n", "\\n").encode()


def array_literal(elems) -> str:
    return "{" + ",".join('"' + e.replace("\\", "\\\\").replace('"', '\\"') + '"' for e in elems) + "}"


def test_heap_resident_text(gpu, oracle_mod):
    """a field that needed unescaping is a heap copy (ETL_COPY_VAL_IN_HEAP): escaped text and jsonb fields, and text[] /
    jsonb[] whose elements carry escapes, next to plain spans and NULLs"""
    oids = [INT4, TEXT, JSONB, 1009, 3807]
    kinds = kinds_of(oracle_mod, oids)
    assert kinds[3] & 0x20 and kinds[4] & 0x20
    texts = ["tab\there back\\slash", "line\nbreak", "plain", "caf\u00e9 \\N", ""]
    docs = ['{"k": "x\\ny",\t"z": [1, "a\\\\b"]}', '{"b":1,\n"a":"\\u00e9"}', '[1.50, "q\\"x"]', '{"plain": true}']
    rows = []
    for r in range(64):
        f = [str(r), copy_escape(texts[r % len(texts)]).decode(), copy_escape(docs[r % len(docs)]).decode(),
             copy_escape(array_literal([texts[(r + k) % len(texts)] for k in range(r % 4)])).decode(),
             copy_escape(array_literal([docs[(r + k) % len(docs)] for k in range(1 + r % 3)])).decode()]
        if r % 7 == 3:
            f[1 + r % 4] = "\\N"
        rows.append(("\t".join(f) + "\n").encode())
    lib = abi.load()
    dec = gpu.Decoder(0)
    dec.put_table_schema(7, cols_of(oids))
    with copy_batch(gpu, dec, 7, rows) as bh:
        p = bh.planes(True)
        tags = np.ctypeslib.as_array(C.cast(p.cell_tag, abi.u8p), shape=(int(p.n_cells),))
        vals = np.ctypeslib.as_array(C.cast(p.cell_val, abi.u64p), shape=(int(p.n_cells),))
        in_heap = (vals >> np.uint64(63)) == 1
        assert in_heap[1::5].sum() > 20 and in_heap[2::5].sum() > 20          # escaped text and jsonb cells
        assert (in_heap[1::5] & (tags[1::5] == 2)).any() and (~in_heap[1::5] & (tags[1::5] == 2)).any()
        want = oracle_rows(oracle_mod, oids, rows)
        assert len(want) == len(rows)
        assert check_copy_emit(lib, bh, kinds, want, "heap text") == len(rows)
    dec.close()


def test_copy_batch_edges(gpu, oracle_mod):
    oids = [INT4, TEXT, JSONB, 1009]
    kinds = kinds_of(oracle_mod, oids)
    lib = abi.load()
    dec = gpu.Decoder(0)
    dec.put_table_schema(7, cols_of(oids))
    with copy_batch(gpu, dec, 7, []) as bh:                       # a 0-row batch
        assert check_copy_emit(lib, bh, kinds, [], "0 rows") == 0
    rows = [b"1\ta\\tb\t{\"k\": 1}\t{x,y}\n", b"2\t\\N\t[]\t\\N\n"]
    with copy_batch(gpu, dec, 7, rows) as bh:
        a = C.c_void_p()
        assert lib.etl_dec_arrow_emit(bh._h, 1, 1, 1, C.byref(a)) == ERR_INVALID_ARG
        # a COPY batch has no schema entries
        s, si = bh.summary(), abi.SchemaInfo()
        assert s.n_schemas == 0 and lib.etl_dec_batch_schema(bh._h, 0, C.byref(si)) != 0
        # the stored schema changes after the decode: the batch keeps the columns it was decoded with
        dec.put_table_schema(7, cols_of([TEXT, INT4]))
        assert check_copy_emit(lib, bh, kinds, oracle_rows(oracle_mod, oids, rows), "schema changed") == 2
    dec.close()


# ------------------------------------------------------------------------------------------------ streaming batches
def decode_stream(gpu, oracle_mod, tables, raw, orc=None, dec=None, carry=None, gpu_carry=None):
    orc = orc or oracle_mod.Oracle()
    if dec is None:
        dec = gpu.Decoder(0)
        for tid, cols in tables.items():
            orc.put_table_schema(tid, cols)
            dec.put_table_schema(tid, cols)
    st = gpu.Stager(len(raw) + 64, 2048)
    st.append_framed(raw)
    inp = st.view()
    gpu.Decoder._carry(inp, gpu_carry)
    return orc.decode(raw, carry), orc, dec, st, inp


def check_cdc_streaming(lib, bh, planes, si, kinds, what):
    """emit with and without the bit: user columns byte-identical, the CDC columns against the restatement"""
    plain, cdc = emit(lib, bh, kinds, si), emit(lib, bh, kinds | CDC, si)
    try:
        n = lib.etl_dec_arrow_rows(cdc)
        recs = [r for r, _ in A.selected_rows(planes, si, kinds)]
        assert n == lib.etl_dec_arrow_rows(plain) == len(recs)
        n_cols = lib.etl_dec_arrow_cols(plain)
        assert lib.etl_dec_arrow_cols(cdc) == n_cols + 2 == planes.schemas[si].n_cols + 2
        if n:
            assert np.array_equal(arr(lib.etl_dec_arrow_row_records(cdc, 1), C.c_uint64, np.uint64, n), np.array(recs, dtype=np.uint64))
        for c in range(n_cols):
            assert raw_column(lib, cdc, c, n) == raw_column(lib, plain, c, n), f"{what}: column {c} changed"
        check_cdc(lib, cdc, n_cols, n, planes, recs, what)
        assert lib.etl_dec_arrow_first_skipped(cdc) == lib.etl_dec_arrow_first_skipped(plain) == R.first_skipped(planes, si, kinds)
        return recs
    finally:
        lib.etl_dec_arrow_free(plain)
        lib.etl_dec_arrow_free(cdc)


@pytest.mark.parametrize("name,scale,kinds", [("c2", 0.01, 7), ("c4", 0.002, 7), ("c4", 0.002, 3), ("c5", 0.002, 7)])
def test_cdc_columns_streaming(gpu, oracle_mod, name, scale, kinds):
    w = wl.make(name, scale, n_segments=1)
    stream, _ = w.generate()
    raw = stream.tobytes()
    planes, orc, dec, st, inp = decode_stream(gpu, oracle_mod, w.table_schemas(), raw)
    lib = abi.load()
    n_rows = 0
    with dec.decode_input(inp, to_host=True) as bh:
        for si in range(len(planes.schemas)):
            n_rows += len(check_cdc_streaming(lib, bh, planes, si, kinds, f"{name} version {si}"))
    assert n_rows > 0
    st.close()
    dec.close()


def test_cdc_keys_after_carry_in(gpu, oracle_mod):
    """a batch that starts inside a transaction: its first keys carry the carried-in final LSN"""
    w = wl.make("c2", 0.01, n_segments=1)
    stream, _ = w.generate()
    cut = wl.mid_transaction_cut(stream, stream.nbytes // 2)
    head, tail = stream[:cut].tobytes(), stream[cut:].tobytes()
    p0, orc, dec, st0, inp0 = decode_stream(gpu, oracle_mod, w.table_schemas(), head)
    with dec.decode_input(inp0, to_host=True) as bh:
        co = bh.summary().carry_out
        gpu_carry = (co.in_tx, co.final_lsn, co.next_tx_ordinal)
    assert gpu_carry == p0.carry_out and gpu_carry[0] and gpu_carry[1]
    p1, _, _, st1, inp1 = decode_stream(gpu, oracle_mod, None, tail, orc, dec, p0.carry_out, gpu_carry)
    lib = abi.load()
    with dec.decode_input(inp1, to_host=True) as bh:
        si = int(p1.rec_schema[int(np.flatnonzero(p1.rec_kind == ord("I"))[0])])
        recs = check_cdc_streaming(lib, bh, p1, si, 7, "carried-in batch")
        assert int(p1.rec_commit_lsn[recs[0]]) == gpu_carry[1]
        a = emit(lib, bh, 7 | CDC, si)
        col = abi.ArrowColumn()
        assert lib.etl_dec_arrow_column(a, lib.etl_dec_arrow_cols(a) - 1, 1, C.byref(col)) == 0
        assert bytes((C.c_uint8 * 16).from_address(col.data)) == b"%016x" % gpu_carry[1]
        lib.etl_dec_arrow_free(a)
    st0.close()
    st1.close()
    dec.close()


def test_first_skipped(gpu, oracle_mod):
    """c5 has partial updates (unchanged TOAST values) and key-only deletes (default replica identity); c3 (REPLICA
    IDENTITY FULL, no deletes) has none"""
    lib = abi.load()
    for name, scale in (("c5", 0.002), ("c3", 0.001)):
        w = wl.make(name, scale, n_segments=1)
        stream, _ = w.generate()
        raw = stream.tobytes()
        planes, orc, dec, st, inp = decode_stream(gpu, oracle_mod, w.table_schemas(), raw)
        seen = set()
        with dec.decode_input(inp, to_host=True) as bh:
            for si in range(len(planes.schemas)):
                for kinds in (1, 2, 4, 6, 7, 7 | ALL | CDC):
                    a = emit(lib, bh, kinds, si)
                    got = lib.etl_dec_arrow_first_skipped(a)
                    lib.etl_dec_arrow_free(a)
                    want = R.first_skipped(planes, si, kinds)
                    assert got == want, (name, si, kinds, got, want)
                    if got != NONE:
                        seen.add((kinds & 7, chr(int(planes.rec_kind[got]))))
        if name == "c5":
            assert {(2, "U"), (4, "D")} <= seen, seen
        else:
            assert not seen
        st.close()
        dec.close()
