"""ClickHouse RowBinary emitter (csrc/rowbinary_emit.cu) against the Python restatement of the ClickHouse destination's
encoding (tests/clickhouse_ref.py) evaluated on the ORACLE's planes: row records, row offsets, every byte and the three
issue reports, for the named workloads, key-only deletes, a hand-built stream of every type, COPY batches, data errors
and the argument checks."""
import ctypes as C

import numpy as np
import pytest

import arrow_ref as A
import clickhouse_ref as R
import scenarios as sc
from canon import decode_cell
from etl_b200 import abi, pgoutput as pg, workloads as wl
from test_gpu_arrow_copy import copy_batch
from test_gpu_arrow_formatted import DOCS, NUMERICS, _big_doc, arr, bits, decode
from test_gpu_copy import REF_ROWS, cols_of, synth_rows

pytestmark = pytest.mark.gpu

ERR_INVALID_ARG = 1
FIXED = {1: 1, 3: 2, 4: 4, 5: 4, 7: 4, 10: 4, 6: 8, 8: 8, 12: 8, 13: 8, 14: 16}


@pytest.fixture(scope="module")
def gpu():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from etl_b200 import decoder
    return decoder


def rb_emit(lib, bh, si, flags, to_host=1):
    fl = (C.c_uint8 * max(1, len(flags)))(*[1 if f else 0 for f in flags])
    h = C.c_void_p()
    rc = lib.etl_dec_rowbinary_emit(bh._h, si, fl, len(flags), to_host, C.byref(h))
    return rc, h


def issue(x):
    return None if x.row == R.NONE64 else (x.row, x.column, x.element)


def fetch(lib, h):
    n = lib.etl_dec_rowbinary_rows(h)
    nbytes = lib.etl_dec_rowbinary_bytes(h)
    offs = arr(lib.etl_dec_rowbinary_row_offsets(h, 1), C.c_uint64, np.uint64, n + 1).copy()   # outlives the emit
    recs = arr(lib.etl_dec_rowbinary_row_records(h, 1), C.c_uint64, np.uint64, n).copy()
    data = bytes((C.c_uint8 * nbytes).from_address(lib.etl_dec_rowbinary_data(h, 1))) if nbytes else b""
    iss = abi.RowBinaryIssues()
    assert lib.etl_dec_rowbinary_issues(h, C.byref(iss)) == 0
    return n, offs, recs, data, iss


def check(lib, h, want, what):
    n, offs, recs, data, iss = fetch(lib, h)
    assert n == len(want["rows"]), (what, n, len(want["rows"]))
    assert np.array_equal(recs, np.array(want["records"], dtype=np.uint64)), what
    want_offs = np.zeros(n + 1, dtype=np.uint64)
    want_offs[1:] = np.cumsum([len(r) for r in want["rows"]])
    if not np.array_equal(offs, want_offs):
        i = int(np.nonzero(offs != want_offs)[0][0])
        raise AssertionError(f"{what}: row offsets differ at {i}: {offs[max(0, i - 1):i + 2]} vs {want_offs[max(0, i - 1):i + 2]}")
    if data != b"".join(want["rows"]):
        i = next(k for k in range(n) if data[offs[k]:offs[k + 1]] != want["rows"][k])
        raise AssertionError(f"{what}: row {i}: {data[offs[i]:offs[i + 1]][:160]!r} != {want['rows'][i][:160]!r}")
    assert issue(iss.date_range) == want["date"], (what, issue(iss.date_range), want["date"])
    assert issue(iss.null_value) == want["null"], (what, issue(iss.null_value), want["null"])
    assert iss.first_partial_update == want["partial"], (what, iss.first_partial_update, want["partial"])
    return n, data, offs


def flag_sets(p, si):
    s = p.schemas[si]
    kinds, cf = [int(k) for k in s.col_kind], [int(f) for f in s.col_flags]
    return {"create_table": R.create_table_flags(kinds, cf), "all": [True] * (s.n_cols + 2)}


def check_streaming(lib, bh, planes, raw, tables, si, flags, what):
    want = R.expected_rowbinary(planes, raw, si, flags, tables[planes.schemas[si].table_id])
    rc, h = rb_emit(lib, bh, si, flags)
    assert rc == 0, (what, rc)
    try:
        return check(lib, h, want, what)
    finally:
        lib.etl_dec_rowbinary_free(h)


# ------------------------------------------------------------------------------------------------ workloads
@pytest.mark.parametrize("name,scale", [("c1", 0.01), ("c2", 0.0005), ("c3", 0.001), ("c4", 0.002), ("c5", 0.0005)])
def test_workloads_match_restatement(gpu, oracle_mod, name, scale):
    w = wl.make(name, scale, n_segments=1)
    stream, _ = w.generate()
    raw = stream.tobytes()
    tables = w.table_schemas()
    planes, dec, st = decode(gpu, oracle_mod, tables, raw)
    lib = abi.load()
    total = 0
    with dec.decode_input(st.view(), to_host=True) as bh:
        for si in range(len(planes.schemas)):
            for fname, flags in flag_sets(planes, si).items():
                n, _, _ = check_streaming(lib, bh, planes, raw, tables, si, flags, f"{name} schema {si} flags {fname}")
                total += n
    assert total > 0
    st.close()
    dec.close()


def test_c5_key_deletes_and_partial_updates_present(gpu, oracle_mod):
    """the c5 stream exercises both the key-image expansion and the partial-update report"""
    w = wl.make("c5", 0.0005, n_segments=1)
    stream, _ = w.generate()
    raw = stream.tobytes()
    tables = w.table_schemas()
    planes, dec, st = decode(gpu, oracle_mod, tables, raw)
    lib = abi.load()
    n = planes.n_records if planes.first_error[0] is None else planes.first_error[0]
    kinds, flags = planes.rec_kind[:n], planes.rec_flags[:n]
    assert ((kinds == ord("D")) & ((flags & 2) != 0)).any()
    partial = [int(r) for r in np.flatnonzero((kinds == ord("U")) & ((flags & 4) != 0) & ((flags & 0x80) != 0))]
    assert partial
    seen = set()
    with dec.decode_input(st.view(), to_host=True) as bh:
        for si in range(len(planes.schemas)):
            rc, h = rb_emit(lib, bh, si, [True] * (planes.schemas[si].n_cols + 2))
            assert rc == 0
            iss = abi.RowBinaryIssues()
            lib.etl_dec_rowbinary_issues(h, C.byref(iss))
            mine = [r for r in partial if int(planes.rec_schema[r]) == si]
            assert iss.first_partial_update == (min(mine) if mine else R.NONE64)
            if mine:
                seen.add(iss.first_partial_update)
            lib.etl_dec_rowbinary_free(h)
    assert min(partial) in seen
    st.close()
    dec.close()


# ------------------------------------------------------------------------------------------------ hand-built streams
SCALARS = [  # (oid, values in text form)
    (16, ["t", "f"]), (21, ["-32768", "32767", "0"]), (23, ["-1", "2147483647"]), (20, ["-9223372036854775808", "42"]),
    (26, ["4294967295", "0"]), (700, ["NaN", "-0", "Infinity", "1.5", "-Infinity"]), (701, ["-0", "NaN", "0", "-Infinity", "2.5e-300"]),
    (1082, ["1969-12-31", "1900-01-01", "2299-12-31", "2024-02-29"]),
    (1083, ["00:00:00", "12:34:56.5", "01:02:03.123456", "23:59:60", "23:59:60.25", "10:00:00.001"]),
    (1114, ["1969-07-20 20:17:40.5", "1900-01-01 00:00:00.000001", "2024-01-02 03:04:05"]),
    (1184, ["1969-12-31 23:59:59.999999+00", "2024-06-01 12:00:00.5-07"]),
    (2950, ["a0eebc99-9c0b-4ef8-bb6d-6bb9bd380a11", "550e8400-e29b-41d4-a716-446655440000"]),
    (17, ["\\x0102ff", "\\x", "\\x" + "ab" * 100]),
    (25, ["", "é✓", "x" * 128, "y" * 16384, "z" * 127]),
]


def hand_built(oracle_mod):
    from test_gpu_parity import ARRAY_COLS
    usable = [(oid, v) for oid, v, _ in ARRAY_COLS if oracle_mod.kind_for_oid(oid) & 0x20]
    cols = [sc.col("id", sc.INT8, 1), sc.col("n", sc.NUMERIC, None, True), sc.col("j", sc.JSONB, None, True), sc.col("j2", 114, None, True)]
    cols += [sc.col(f"s{oid}", oid, None, True) for oid, _ in SCALARS] + [sc.col(f"a{oid}", oid, None, True) for oid, _ in usable]
    docs = DOCS + [_big_doc()]

    def row(r):
        vals = [str(r), NUMERICS[r % len(NUMERICS)] if r % 11 else None, docs[r % len(docs)] if r % 9 else None, docs[(r * 7) % len(docs)]]
        vals += [None if (r + j) % 13 == 0 else v[(r + j) % len(v)] for j, (_, v) in enumerate(SCALARS)]
        for j, (_, v) in enumerate(usable):
            k = (r + j) % (len(v) + 2)
            vals.append(None if k == len(v) else ("{}" if k == len(v) + 1 else v[k]))
        return vals
    return cols, row, 3 * len(docs) * 4


def test_hand_built_stream(gpu, oracle_mod):
    """every scalar type and array element kind with NULLs and empty arrays; Numeric specials, Json escapes, duplicate
    keys and a >= 256 KiB document; Time fractions and the leap second; pre-1970 timestamps; Float NaN / +-0; strings
    whose varints take 2 and 3 bytes; date[] with 0001-01-01 (a Date32 issue inside an array).  Both flag sets, and the
    Numeric / Json text equals the Arrow ALL_COLUMNS text of the same rows."""
    cols, row, n_rows = hand_built(oracle_mod)
    rel = pg.relation(95, "public", "rb", "f", sc.rel_cols(cols, set()))
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
    raw = w.bytes()
    tables = {95: cols}
    planes, dec, st = decode(gpu, oracle_mod, tables, raw)
    assert planes.first_error[0] is None, planes.first_error
    lib = abi.load()
    kinds = [int(k) for k in planes.schemas[0].col_kind]
    with dec.decode_input(st.view(), to_host=True) as bh:
        for fname, flags in flag_sets(planes, 0).items():
            n, data, offs = check_streaming(lib, bh, planes, raw, tables, 0, flags, f"hand-built {fname}")
            assert n > 0
        # the Numeric / Json text inside the RowBinary (all flags set) equals the Arrow ALL_COLUMNS text
        a = C.c_void_p()
        assert lib.etl_dec_arrow_emit(bh._h, 0, 7 | A.ALL_COLUMNS, 1, C.byref(a)) == 0
        try:
            assert lib.etl_dec_arrow_rows(a) == n
            rows = [split_row(data[offs[i]:offs[i + 1]], kinds + [2, 6], [True] * (len(kinds) + 2)) for i in range(n)]
            n_cross = 0
            for c in (1, 2, 3):
                col = abi.ArrowColumn()
                assert lib.etl_dec_arrow_column(a, c, 1, C.byref(col)) == 0
                aoffs = arr(col.offsets, C.c_int32, np.int32, n + 1)
                valid = bits(col.validity, n)
                text = bytes((C.c_uint8 * col.data_bytes).from_address(col.data))
                for i in range(n):
                    got = rows[i][c]
                    assert (got is not None) == bool(valid[i]), (c, i)
                    if got is not None:
                        assert strip_varint(got) == text[aoffs[i]:aoffs[i + 1]], (c, i)
                        n_cross += 1
            assert n_cross > n
        finally:
            lib.etl_dec_arrow_free(a)
    st.close()
    dec.close()


def read_varint(b, pos):
    v, shift = 0, 0
    while True:
        x = b[pos]
        pos += 1
        v |= (x & 0x7F) << shift
        shift += 7
        if not x & 0x80:
            return v, pos


def strip_varint(b):
    n, pos = read_varint(b, 0)
    assert pos + n == len(b)
    return b[pos:]


def skip_value(k, b, pos):
    if k & 0x20:
        n, pos = read_varint(b, pos)
        for _ in range(n):
            pos += 1
            if b[pos - 1] == 0:
                pos = skip_value(k & 0x1F, b, pos)
        return pos
    if k in FIXED:
        return pos + FIXED[k]
    n, pos = read_varint(b, pos)
    return pos + n


def split_row(b, kinds, flags):
    """one RowBinary row → the value bytes of each column (None for NULL), by the column classes"""
    pos, out = 0, []
    for k, f in zip(kinds, flags):
        if f:
            pos += 1
            if b[pos - 1] == 1:
                out.append(None)
                continue
        start = pos
        pos = skip_value(k, b, pos)
        out.append(b[start:pos])
    assert pos == len(b)
    return out


KEY_COLS = [sc.col("id", sc.INT8, 1), sc.col("k2", sc.TEXT, 2)] + \
    [sc.col(f"nn{oid}", oid) for oid in (16, 21, 23, 20, 26, 700, 701, 1700, 1082, 1083, 1114, 1184, 2950, 114, 3802, 17, 25, 1007, 1009)] + \
    [sc.col(f"nl{oid}", oid, None, True) for oid in (23, 25, 1082, 1007)]


def key_row(r):
    vals = [str(r), f"k{r}", "t", "7", "8", "9", "10", "1.5", "2.5", "3.5", "2024-01-02", "01:02:03", "2024-01-02 03:04:05",
            "2024-01-02 03:04:05+00", "a0eebc99-9c0b-4ef8-bb6d-6bb9bd380a11", '{"a":1}', '{"b":2}', "\\x01", "t", "{1}", "{a}"]
    return vals + [None if r % 2 else "5", "s", "2024-01-01", "{2}"]


def test_key_only_deletes(gpu, oracle_mod):
    """REPLICA IDENTITY DEFAULT: deletes carry the key image only; non-key columns of every class become NULL (nullable
    scalars) or default_cell's zero bytes (NOT NULL columns and arrays); with create-table flags a NULL lands in a
    nullable column, with no flags set every NULL is a reported issue"""
    rel = pg.relation(96, "public", "keys", "d", sc.rel_cols(KEY_COLS, {"id", "k2"}))
    w = pg.StreamWriter()
    tx = sc.Tx(w)
    tx.begin()
    w.emit(rel)
    for r in range(300):
        w.emit(pg.insert(96, key_row(r)))
        if r % 2:
            w.emit(pg.delete(96, key=[str(r), f"k{r}"]))
    tx.commit()
    raw = w.bytes()
    tables = {96: KEY_COLS}
    planes, dec, st = decode(gpu, oracle_mod, tables, raw)
    assert planes.first_error[0] is None, planes.first_error
    assert ((planes.rec_flags[:planes.n_records] & 2) != 0).sum() == 150
    lib = abi.load()
    nc = planes.schemas[0].n_cols
    with dec.decode_input(st.view(), to_host=True) as bh:
        for fname, flags in list(flag_sets(planes, 0).items()) + [("none", [False] * (nc + 2))]:
            check_streaming(lib, bh, planes, raw, tables, 0, flags, f"key deletes {fname}")
    st.close()
    dec.close()


def test_date_out_of_range_and_null_under_cleared_flag(gpu, oracle_mod):
    """a Date out of Date32's range as a scalar and inside a date[], a NULL in a column without the Nullable flag: the
    first of each is reported, the rows before it are exact"""
    cols = [sc.col("id", sc.INT8, 1), sc.col("d", sc.DATE, None, True), sc.col("da", 1182, None, True), sc.col("t", sc.TEXT, None, True)]
    rel = pg.relation(97, "public", "dates", "f", sc.rel_cols(cols, set()))
    w = pg.StreamWriter()
    tx = sc.Tx(w)
    tx.begin()
    w.emit(rel)
    for r in range(200):
        d = "1899-12-31" if r == 150 else ("2300-01-01" if r == 170 else "2000-01-01")
        da = "{2000-01-01,NULL,0001-01-01}" if r == 120 else "{2000-01-01}"
        w.emit(pg.insert(97, [str(r), d, da, None if r in (90, 95) else "x"]))
    tx.commit()
    raw = w.bytes()
    tables = {97: cols}
    planes, dec, st = decode(gpu, oracle_mod, tables, raw)
    assert planes.first_error[0] is None, planes.first_error
    lib = abi.load()
    with dec.decode_input(st.view(), to_host=True) as bh:
        _, _, _ = check_streaming(lib, bh, planes, raw, tables, 0, [True] * 6, "all flags")
        rc, h = rb_emit(lib, bh, 0, [True, True, True, False, False, False])
        assert rc == 0
        n, offs, _, _, iss = fetch(lib, h)
        assert issue(iss.date_range) == (120, 2, 2)
        assert issue(iss.null_value) == (90, 3, R.NONE32)
        lib.etl_dec_rowbinary_free(h)
        check_streaming(lib, bh, planes, raw, tables, 0, [True, False, True, False, False, False], "cleared flags")
    st.close()
    dec.close()


# ------------------------------------------------------------------------------------------------ COPY batches
def copy_want(oracle_mod, oids, rows, flags):
    cells = []
    for row in rows:
        e, _, cs, text, heap = oracle_mod.parse_copy_row(oids, row)
        if e:
            break
        cells.append([(t, decode_cell(t, v, a, text, heap)) for t, v, a in cs])
    return R.expected_copy_rowbinary(cells, flags)


@pytest.mark.parametrize("idx", range(len(REF_ROWS)))
def test_copy_reference_vectors(gpu, oracle_mod, idx):
    """table_row.rs:206-533, each as a one-row batch; an erroring vector gives zero rows"""
    oids, row = REF_ROWS[idx]
    lib = abi.load()
    dec = gpu.Decoder(0)
    dec.put_table_schema(7, cols_of(oids))
    with copy_batch(gpu, dec, 7, [row]) as bh:
        for flags in ([True] * (len(oids) + 2), [False] * (len(oids) + 2)):
            rc, h = rb_emit(lib, bh, 0, flags)
            assert rc == 0
            check(lib, h, copy_want(oracle_mod, oids, [row], flags), f"vector {idx}")
            lib.etl_dec_rowbinary_free(h)
        rc, h = rb_emit(lib, bh, 1, [True] * (len(oids) + 2))
        assert rc == ERR_INVALID_ARG
    dec.close()


@pytest.mark.parametrize("n,bad_at", [(5000, 3777), (200000, None)])
def test_copy_synthetic_tables(gpu, oracle_mod, n, bad_at):
    """rows with NULLs, escapes that needed unescaping (heap text) and non-ASCII text; a mid-batch parse error"""
    oids, rows = synth_rows(n, 1234 + n, bad_at)
    lib = abi.load()
    dec = gpu.Decoder(0)
    dec.put_table_schema(7, cols_of(oids))
    flags = [True] * len(oids) + [False, False]
    with copy_batch(gpu, dec, 7, rows) as bh:
        want = copy_want(oracle_mod, oids, rows, flags)
        assert len(want["rows"]) == (bad_at if bad_at is not None else n)
        for to_host in (1, 0):
            rc, h = rb_emit(lib, bh, 0, flags, to_host)
            assert rc == 0
            if to_host:
                check(lib, h, want, f"copy {n}")
            else:
                assert lib.etl_dec_rowbinary_data(h, 1) is None and lib.etl_dec_rowbinary_data(h, 0)
                assert lib.etl_dec_rowbinary_bytes(h) == sum(len(r) for r in want["rows"])
            lib.etl_dec_rowbinary_free(h)
    dec.close()


# ------------------------------------------------------------------------------------------------ errors, arguments, lifetime
def test_mid_batch_decode_error_and_arguments(gpu, oracle_mod):
    cols = [sc.col("id", sc.INT8, 1), sc.col("n", sc.NUMERIC, None, True), sc.col("j", sc.JSONB, None, True), sc.col("a", 1231, None, True)]
    rel = pg.relation(94, "public", "err", "d", sc.rel_cols(cols, {"id"}))
    w = pg.StreamWriter()
    tx = sc.Tx(w)
    tx.begin()
    w.emit(rel)
    for r in range(40):
        w.emit(pg.insert(94, [str(r), "%d.5" % r if r != 23 else "1.2.3", '{"r":%d,"a":[%d]}' % (r, r), "{%d,NULL,1.50}" % r]))
    tx.commit()
    raw = w.bytes()
    tables = {94: cols}
    planes, dec, st = decode(gpu, oracle_mod, tables, raw)
    assert planes.first_error[0] is not None
    lib = abi.load()
    with dec.decode_input(st.view(), to_host=True) as bh:
        n, _, _ = check_streaming(lib, bh, planes, raw, tables, 0, [True] * 6, "mid-batch error")
        assert n == 23
        for nf in (0, 5, 7):
            assert rb_emit(lib, bh, 0, [True] * nf)[0] == ERR_INVALID_ARG
        assert rb_emit(lib, bh, len(planes.schemas), [True] * 6)[0] == ERR_INVALID_ARG
    st.close()
    dec.close()


def test_zero_row_emit(gpu, oracle_mod):
    cols = [sc.col("id", sc.INT8, 1), sc.col("t", sc.TEXT, None, True)]
    w = pg.StreamWriter()
    tx = sc.Tx(w)
    tx.begin()
    w.emit(pg.relation(98, "public", "empty", "d", sc.rel_cols(cols, {"id"})))
    tx.commit()
    raw = w.bytes()
    planes, dec, st = decode(gpu, oracle_mod, {98: cols}, raw)
    lib = abi.load()
    with dec.decode_input(st.view(), to_host=True) as bh:
        rc, h = rb_emit(lib, bh, 0, [True] * 4)
        assert rc == 0
        check(lib, h, dict(records=[], rows=[], date=None, null=None, partial=R.NONE64), "empty")
        assert lib.etl_dec_rowbinary_bytes(h) == 0
        lib.etl_dec_rowbinary_free(h)
    st.close()
    dec.close()


def test_emit_free_cycles_keep_memory_stable(gpu, oracle_mod):
    cols, row, n_rows = hand_built(oracle_mod)
    w = pg.StreamWriter()
    tx = sc.Tx(w)
    tx.begin()
    w.emit(pg.relation(95, "public", "rb", "f", sc.rel_cols(cols, set())))
    for r in range(n_rows):
        w.emit(pg.insert(95, row(r)))
    tx.commit()
    raw = w.bytes()
    planes, dec, st = decode(gpu, oracle_mod, {95: cols}, raw)
    lib = abi.load()
    flags = [True] * (len(cols) + 2)
    free, total = C.c_uint64(), C.c_uint64()
    with dec.decode_input(st.view(), to_host=True) as bh:
        first = None
        for i in range(100):
            rc, h = rb_emit(lib, bh, 0, flags, to_host=1 - i % 2)
            assert rc == 0
            if first is None:
                first = fetch(lib, h)[3]
            lib.etl_dec_rowbinary_free(h)
            assert lib.etl_dec_mem_info(dec._ctx, C.byref(free), C.byref(total)) == 0
            if i == 1:
                base = free.value
        assert abs(free.value - base) <= 4 << 20, (free.value, base)
        assert first
    st.close()
    dec.close()
