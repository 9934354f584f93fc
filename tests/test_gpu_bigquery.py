"""BigQuery Storage Write emitter (csrc/bigquery_emit.cu) against the Python restatement of the BigQuery destination's
rows (tests/bigquery_ref.py) evaluated on the ORACLE's planes: row records, row offsets, every byte, the first value
issue and the first invalid record, for the named workloads, hand-built streams of every type and of the key-change
cases, COPY batches, data errors and the argument checks.  Every emitted row is also parsed with a small protobuf wire
reader and checked field by field."""
import ctypes as C

import numpy as np
import pytest

import arrow_ref as A
import bigquery_ref as R
import scenarios as sc
from canon import decode_cell
from etl_b200 import abi, pgoutput as pg, workloads as wl
from test_gpu_arrow_copy import copy_batch
from test_gpu_arrow_formatted import arr, bits, decode
from test_gpu_copy import REF_ROWS, cols_of, synth_rows
from test_gpu_rowbinary import hand_built

pytestmark = pytest.mark.gpu

ERR_INVALID_ARG = 1


@pytest.fixture(scope="module")
def gpu():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from etl_b200 import decoder
    return decoder


def bq_emit(lib, bh, si, to_host=1):
    h = C.c_void_p()
    rc = lib.etl_dec_bigquery_emit(bh._h, si, to_host, C.byref(h))
    return rc, h


def fetch(lib, h):
    n = lib.etl_dec_bigquery_rows(h)
    nbytes = lib.etl_dec_bigquery_bytes(h)
    offs = arr(lib.etl_dec_bigquery_row_offsets(h, 1), C.c_uint64, np.uint64, n + 1).copy()
    recs = arr(lib.etl_dec_bigquery_row_records(h, 1), C.c_uint64, np.uint64, n).copy()
    data = bytes((C.c_uint8 * nbytes).from_address(lib.etl_dec_bigquery_data(h, 1))) if nbytes else b""
    iss = abi.BigQueryIssues()
    assert lib.etl_dec_bigquery_issues(h, C.byref(iss)) == 0
    return n, offs, recs, data, iss


def value_issue(x):
    return None if x.row == R.NONE64 else (x.row, x.column, x.element, x.kind)


# ------------------------------------------------------------------------------------------------ wire reader
def read_varint(b, pos):
    v, shift = 0, 0
    while True:
        x = b[pos]
        pos += 1
        v |= (x & 0x7F) << shift
        shift += 7
        if not x & 0x80:
            return v, pos


def parse_message(b):
    """protobuf wire format → [(field, wire type, value bytes or int)]"""
    pos, out = 0, []
    while pos < len(b):
        k, pos = read_varint(b, pos)
        field, wt = k >> 3, k & 7
        if wt == 0:
            v, pos = read_varint(b, pos)
        elif wt == 1:
            v, pos = b[pos:pos + 8], pos + 8
        elif wt == 5:
            v, pos = b[pos:pos + 4], pos + 4
        elif wt == 2:
            n, pos = read_varint(b, pos)
            v, pos = b[pos:pos + n], pos + n
        else:
            raise AssertionError(f"wire type {wt}")
        out.append((field, wt, v))
    assert pos == len(b)
    return out


def check_fields(rows, n_cols, streaming):
    """every row parses; field numbers ascend (repeated fields stay together); _CHANGE_TYPE / sequence are present"""
    for i, row in enumerate(rows):
        fields = parse_message(row)
        nums = [f for f, _, _ in fields]
        assert nums == sorted(nums), i
        assert (n_cols + 1, 2, b"UPSERT") in fields or (n_cols + 1, 2, b"DELETE") in fields, i
        seq = [v for f, _, v in fields if f == n_cols + 2]
        if streaming:
            assert len(seq) == 1 and len(seq[0]) == 50 and seq[0].count(b"/") == 2, i
        else:
            assert not seq
        assert all(1 <= f <= n_cols + 2 for f in nums)


def check(lib, h, want, what, n_cols, streaming=True):
    n, offs, recs, data, iss = fetch(lib, h)
    assert n == len(want["rows"]), (what, n, len(want["rows"]))
    assert np.array_equal(recs, np.array(want["records"], dtype=np.uint64)), what
    want_offs = np.zeros(n + 1, dtype=np.uint64)
    want_offs[1:] = np.cumsum([len(r) for r in want["rows"]])
    if not np.array_equal(offs, want_offs):
        i = int(np.nonzero(offs != want_offs)[0][0])
        raise AssertionError(f"{what}: row offsets differ at {i}: {offs[max(0, i - 1):i + 2]} vs {want_offs[max(0, i - 1):i + 2]}")
    assert value_issue(iss.value) == want["value"], (what, value_issue(iss.value), want["value"])
    assert iss.first_invalid_record == want["invalid"], (what, iss.first_invalid_record, want["invalid"])
    # the rows of this emitter are exact throughout (a NULL array element writes nothing), not only before the issue
    exact = n
    for i in range(exact):
        got = data[offs[i]:offs[i + 1]]
        if got != want["rows"][i]:
            raise AssertionError(f"{what}: row {i}: {got[:200]!r} != {want['rows'][i][:200]!r}")
    check_fields([data[offs[i]:offs[i + 1]] for i in range(exact)], n_cols, streaming)
    return n, data, offs


def check_streaming(lib, bh, planes, raw, tables, si, what):
    want = R.expected_bigquery(planes, raw, si, tables[planes.schemas[si].table_id])
    rc, h = bq_emit(lib, bh, si)
    assert rc == 0, (what, rc)
    try:
        return check(lib, h, want, what, planes.schemas[si].n_cols) + (want,)
    finally:
        lib.etl_dec_bigquery_free(h)


def run_stream(gpu, oracle_mod, tables, raw, what, first_error_ok=False):
    planes, dec, st = decode(gpu, oracle_mod, tables, raw)
    if not first_error_ok:
        assert planes.first_error[0] is None, planes.first_error
    lib = abi.load()
    out = []
    with dec.decode_input(st.view(), to_host=True) as bh:
        for si in range(len(planes.schemas)):
            out.append(check_streaming(lib, bh, planes, raw, tables, si, f"{what} schema {si}"))
    st.close()
    dec.close()
    return planes, out


# ------------------------------------------------------------------------------------------------ workloads
@pytest.mark.parametrize("name,scale", [("c1", 0.01), ("c2", 0.0005), ("c3", 0.001), ("c4", 0.002), ("c5", 0.0005)])
def test_workloads_match_restatement(gpu, oracle_mod, name, scale):
    w = wl.make(name, scale, n_segments=1)
    stream, _ = w.generate()
    raw = stream.tobytes()
    planes, out = run_stream(gpu, oracle_mod, w.table_schemas(), raw, name, first_error_ok=True)
    assert sum(o[0] for o in out) > 0


# ------------------------------------------------------------------------------------------------ hand-built streams
def test_hand_built_every_kind(gpu, oracle_mod):
    """every scalar type and array element kind (NULLs, empty arrays, Numeric specials, Json escapes and a large
    document, Time fractions, pre-1970 timestamps, Float NaN / -0) as inserts, FULL-identity updates that change the
    key (DELETE + UPSERT) and deletes; the Numeric / Json text of the UPSERT rows equals the Arrow ALL_COLUMNS text"""
    cols, row, n_rows = hand_built(oracle_mod)
    rel = pg.relation(95, "public", "bq", "f", sc.rel_cols(cols, set()))
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
    lib = abi.load()
    with dec.decode_input(st.view(), to_host=True) as bh:
        n, data, offs, want = check_streaming(lib, bh, planes, raw, tables, 0, "hand-built")
        assert n > 0
        # Numeric (column 1) and Json (2, 3) text of the UPSERT rows against the Arrow ALL_COLUMNS text of the same images
        a = C.c_void_p()
        assert lib.etl_dec_arrow_emit(bh._h, 0, 3 | A.ALL_COLUMNS, 1, C.byref(a)) == 0
        try:
            upserts = [i for i in range(n) if (len(cols) + 1, 2, b"UPSERT") in parse_message(data[offs[i]:offs[i + 1]])]
            assert lib.etl_dec_arrow_rows(a) == len(upserts)
            n_cross = 0
            for c in (1, 2, 3):
                col = abi.ArrowColumn()
                assert lib.etl_dec_arrow_column(a, c, 1, C.byref(col)) == 0
                m = len(upserts)
                aoffs = arr(col.offsets, C.c_int32, np.int32, m + 1)
                valid = bits(col.validity, m)
                text = bytes((C.c_uint8 * col.data_bytes).from_address(col.data))
                for k, i in enumerate(upserts):
                    got = [v for f, _, v in parse_message(data[offs[i]:offs[i + 1]]) if f == c + 1]
                    assert (len(got) == 1) == bool(valid[k]), (c, i)
                    if got:
                        assert got[0] == text[aoffs[k]:aoffs[k + 1]], (c, i)
                        n_cross += 1
            assert n_cross > len(upserts)
        finally:
            lib.etl_dec_arrow_free(a)
    st.close()
    dec.close()


def _key_stream(rel_id, cols, identity, key_names, events):
    w = pg.StreamWriter()
    tx = sc.Tx(w)
    tx.begin()
    w.emit(pg.relation(rel_id, "public", f"k{rel_id}", identity, sc.rel_cols(cols, key_names)))
    for e in events:
        w.emit(e)
    tx.commit()
    return w.bytes()


def test_key_changes_under_full_identity(gpu, oracle_mod):
    """composite primary key (int8, text) under REPLICA IDENTITY FULL: an unchanged key gives one UPSERT, a change in
    either column gives DELETE (ordinal 0, key columns only) + UPSERT (ordinal 1); a NaN float key always changes,
    -0 equals +0, a Numeric 1.0 → 1.00 changes, a jsonb key with its members reordered does not"""
    cols = [sc.col("a", sc.INT8, 1), sc.col("b", sc.TEXT, 2), sc.col("f", 701, 3), sc.col("n", sc.NUMERIC, 4),
            sc.col("j", sc.JSONB, 5), sc.col("v", sc.TEXT, None, True)]
    base = ["1", "x" * 100, "1.5", "1.0", '{"a":1,"b":[1,2]}', "v"]
    ev = []
    for r in range(40):
        old = list(base)
        old[0] = str(r)
        new = list(old)
        m = r % 8
        if m == 1:
            new[1] = "x" * 99 + "y"               # long text key changes in its last byte
        elif m == 2:
            old[2] = new[2] = "NaN"
        elif m == 3:
            old[2], new[2] = "-0", "0"
        elif m == 4:
            new[3] = "1.00"
        elif m == 5:
            new[4] = '{"b":[1,2], "a":1}'
        elif m == 6:
            new[0] = str(r + 1000)
        new[5] = f"v{r}"
        ev.append(pg.insert(90, old))
        ev.append(pg.update(90, new, old=old))
        if r % 4 == 0:
            ev.append(pg.delete(90, old=new))
    raw = _key_stream(90, cols, "f", {"a", "b", "f", "n", "j"}, ev)
    planes, out = run_stream(gpu, oracle_mod, {90: cols}, raw, "full identity")
    n, data, offs, want = out[0]
    deletes = [i for i in range(n) if (len(cols) + 1, 2, b"DELETE") in parse_message(data[offs[i]:offs[i + 1]])]
    # per 8 records: m == 1, 2 (NaN), 4, 6 change the key; plus every 4th record's delete
    assert len(deletes) == 40 // 8 * 4 + 10
    for i in deletes:
        assert all(f <= 5 or f >= 7 for f, _, _ in parse_message(data[offs[i]:offs[i + 1]]))


def test_key_images_and_invalid_records(gpu, oracle_mod):
    """REPLICA IDENTITY DEFAULT: updates that change the key carry a key image (DELETE from it + UPSERT), key-only
    deletes give sparse DELETE rows; partial updates and deletes without an old image are invalid records.  A table
    whose identity index is not its primary key (identity 'i') turns every key image into an invalid record."""
    cols = [sc.col("id", sc.INT8, 1), sc.col("k2", sc.TEXT, 2), sc.col("t", sc.TEXT, None, True), sc.col("big", sc.TEXT, None, True)]
    ev = []
    for r in range(60):
        row = [str(r), f"k{r}", "t", "b" * 300]
        ev.append(pg.insert(91, row))
        if r % 3 == 0:
            ev.append(pg.update(91, [str(r + 500), f"k{r}", "t2", "b"], key=[str(r), f"k{r}"]))
        elif r % 3 == 1:
            ev.append(pg.update(91, [str(r), f"k{r}", "t3", "c"]))
        elif r % 6 == 2:
            ev.append(pg.update(91, [str(r), f"k{r}", "t4", pg.UNCHANGED]))   # partial: an invalid record
        if r % 5 == 0:
            ev.append(pg.delete(91, key=[str(r), f"k{r}"]))
    raw = _key_stream(91, cols, "d", {"id", "k2"}, ev)
    planes, out = run_stream(gpu, oracle_mod, {91: cols}, raw, "key images")
    n, data, offs, want = out[0]
    assert want["invalid"] != R.NONE64
    assert len(want["rows"]) == 60 + 20 * 2 + 20 + 12

    # identity 'i' over column t while the primary key is (id, k2): key images are invalid
    cols_i = [sc.col("id", sc.INT8, 1), sc.col("t", sc.TEXT)]
    ev = [pg.insert(92, ["1", "a"]), pg.update(92, ["1", "b"]), pg.delete(92, key=["b"]), pg.insert(92, ["2", "c"])]
    raw = _key_stream(92, cols_i, "i", {"t"}, ev)
    planes, out = run_stream(gpu, oracle_mod, {92: cols_i}, raw, "identity i")
    assert out[0][3]["invalid"] != R.NONE64


def test_value_issues_at_their_boundaries(gpu, oracle_mod):
    """a NULL inside an array, a Numeric with 38 / 39 fractional digits, Json integers at the i64 / u64 edges: the
    first issue in (row, column) order is reported, the rows before it are exact"""
    cols = [sc.col("id", sc.INT8, 1), sc.col("n", sc.NUMERIC, None, True), sc.col("j", sc.JSONB, None, True),
            sc.col("ia", 1007, None, True), sc.col("na", 1231, None, True), sc.col("ja", 3807, None, True)]
    ok_rows = [
        ["0", "0." + "0" * 37 + "1", '{"a":-9223372036854775808,"b":18446744073709551615,"c":1e400}', "{1,2}", "{1.5}", '{"[1]"}'],
        ["1", "0." + "0" * 50, '[18446744073709551615.0, "99999999999999999999"]', "{}", "{NaN}", None],
    ]

    def build(bad):
        ev = [pg.insert(93, r) for r in ok_rows]
        ev.append(pg.insert(93, bad))
        ev.append(pg.insert(93, ["99", "1", "{}", "{NULL}", None, None]))
        return _key_stream(93, cols, "f", set(), ev)

    cases = [
        (["2", "1", "{}", "{1,NULL,3}", "{0." + "0" * 38 + "1}", None], (2, 3, 1, R.ISSUE_ARRAY_NULL)),
        (["2", "0." + "0" * 38 + "1", "{}", None, None, None], (2, 1, R.NONE32, R.ISSUE_NUMERIC_SCALE)),
        (["2", None, '{"x":[18446744073709551616]}', None, None, None], (2, 2, R.NONE32, R.ISSUE_JSON_INTEGER)),
        (["2", None, '[-9223372036854775809]', None, None, None], (2, 2, R.NONE32, R.ISSUE_JSON_INTEGER)),
        (["2", None, None, None, "{1,0." + "0" * 39 + "1}", None], (2, 4, 1, R.ISSUE_NUMERIC_SCALE)),
        (["2", None, None, None, None, '{"1","[1,-9223372036854775809]"}'], (2, 5, 1, R.ISSUE_JSON_INTEGER)),
    ]
    for bad, want in cases:
        raw = build(bad)
        planes, out = run_stream(gpu, oracle_mod, {93: cols}, raw, f"issue {want}")
        assert out[0][3]["value"] == want, (out[0][3]["value"], want)


# ------------------------------------------------------------------------------------------------ COPY batches
def copy_want(oracle_mod, oids, rows):
    cells = []
    for row in rows:
        e, _, cs, text, heap = oracle_mod.parse_copy_row(oids, row)
        if e:
            break
        cells.append([(t, decode_cell(t, v, a, text, heap)) for t, v, a in cs])
    return R.expected_copy_bigquery(cells)


@pytest.mark.parametrize("idx", range(len(REF_ROWS)))
def test_copy_reference_vectors(gpu, oracle_mod, idx):
    oids, row = REF_ROWS[idx]
    lib = abi.load()
    dec = gpu.Decoder(0)
    dec.put_table_schema(7, cols_of(oids))
    with copy_batch(gpu, dec, 7, [row]) as bh:
        rc, h = bq_emit(lib, bh, 0)
        assert rc == 0
        check(lib, h, copy_want(oracle_mod, oids, [row]), f"vector {idx}", len(oids), streaming=False)
        lib.etl_dec_bigquery_free(h)
        assert bq_emit(lib, bh, 1)[0] == ERR_INVALID_ARG
    dec.close()


@pytest.mark.parametrize("n,bad_at", [(5000, 3777), (200000, None)])
def test_copy_synthetic_tables(gpu, oracle_mod, n, bad_at):
    oids, rows = synth_rows(n, 1234 + n, bad_at)
    lib = abi.load()
    dec = gpu.Decoder(0)
    dec.put_table_schema(7, cols_of(oids))
    with copy_batch(gpu, dec, 7, rows) as bh:
        want = copy_want(oracle_mod, oids, rows)
        assert len(want["rows"]) == (bad_at if bad_at is not None else n)
        for to_host in (1, 0):
            rc, h = bq_emit(lib, bh, 0, to_host)
            assert rc == 0
            if to_host:
                check(lib, h, want, f"copy {n}", len(oids), streaming=False)
            else:
                assert lib.etl_dec_bigquery_data(h, 1) is None and lib.etl_dec_bigquery_data(h, 0)
                assert lib.etl_dec_bigquery_bytes(h) == sum(len(r) for r in want["rows"])
            lib.etl_dec_bigquery_free(h)
    dec.close()


# ------------------------------------------------------------------------------------------------ errors, arguments, lifetime
def test_mid_batch_decode_error_and_arguments(gpu, oracle_mod):
    cols = [sc.col("id", sc.INT8, 1), sc.col("n", sc.NUMERIC, None, True), sc.col("j", sc.JSONB, None, True), sc.col("a", 1231, None, True)]
    ev = [pg.insert(94, [str(r), "%d.5" % r if r != 23 else "1.2.3", '{"r":%d,"a":[%d]}' % (r, r), "{%d,1.50}" % r]) for r in range(40)]
    raw = _key_stream(94, cols, "d", {"id"}, ev)
    tables = {94: cols}
    planes, dec, st = decode(gpu, oracle_mod, tables, raw)
    assert planes.first_error[0] is not None
    lib = abi.load()
    with dec.decode_input(st.view(), to_host=True) as bh:
        n, _, _, _ = check_streaming(lib, bh, planes, raw, tables, 0, "mid-batch error")
        assert n == 23
        assert bq_emit(lib, bh, len(planes.schemas))[0] == ERR_INVALID_ARG
        assert lib.etl_dec_bigquery_emit(bh._h, 0, 1, None) == ERR_INVALID_ARG
    st.close()
    dec.close()


def test_emit_free_cycles_keep_memory_stable(gpu, oracle_mod):
    cols, row, n_rows = hand_built(oracle_mod)
    w = pg.StreamWriter()
    tx = sc.Tx(w)
    tx.begin()
    w.emit(pg.relation(95, "public", "bq", "f", sc.rel_cols(cols, set())))
    for r in range(n_rows):
        w.emit(pg.insert(95, row(r)))
    tx.commit()
    raw = w.bytes()
    planes, dec, st = decode(gpu, oracle_mod, {95: cols}, raw)
    lib = abi.load()
    free, total = C.c_uint64(), C.c_uint64()
    with dec.decode_input(st.view(), to_host=True) as bh:
        first = None
        for i in range(100):
            rc, h = bq_emit(lib, bh, 0, to_host=1 - i % 2)
            assert rc == 0
            if first is None:
                first = fetch(lib, h)[3]
            lib.etl_dec_bigquery_free(h)
            assert lib.etl_dec_mem_info(dec._ctx, C.byref(free), C.byref(total)) == 0
            if i == 1:
                base = free.value
        assert abs(free.value - base) <= 4 << 20, (free.value, base)
        assert first
    st.close()
    dec.close()
