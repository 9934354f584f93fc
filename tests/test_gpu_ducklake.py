"""DuckLake emitter (csrc/ducklake_emit.cu) against the Python restatement of the DuckLake destination
(tests/ducklake_ref.py) evaluated on the ORACLE's planes: mutation kinds and records, the row / predicate / assignment
texts byte for byte with their offsets, the issues, the sub-batches with their fingerprints and batch ids, and the COPY
fingerprint, for the named workloads, hand-built streams of every type, the identity and partial-update cases, Truncate
cuts, COPY batches, data errors and the argument checks.  A Delete without any old image cannot be written by the test
stream writer: only the restatement and the selection rule cover that reject."""
import ctypes as C

import numpy as np
import pytest

import ducklake_ref as R
import scenarios as sc
from canon import decode_cell
from etl_b200 import abi, pgoutput as pg, workloads as wl
from test_gpu_arrow_copy import copy_batch
from test_gpu_arrow_formatted import arr, decode
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


def quote_ident(name: str) -> str:
    """quote_identifier for the names these tests use: quoted unless lowercase letters, digits and _"""
    if name and all(c.islower() or c.isdigit() or c == "_" for c in name) and not name[0].isdigit():
        return name
    return '"' + name.replace('"', '""') + '"'


def dl_emit(lib, bh, si, names, to_host=1):
    arr_t = (C.c_char_p * max(1, len(names)))(*[n.encode() for n in names])
    h = C.c_void_p()
    rc = lib.etl_dec_ducklake_emit(bh._h, si, arr_t, len(names), to_host, C.byref(h))
    return rc, h


def fetch(lib, h):
    n = lib.etl_dec_ducklake_mutations(h)
    kinds = list(arr(lib.etl_dec_ducklake_kinds(h, 1), C.c_uint8, np.uint8, n)) if n else []
    recs = list(arr(lib.etl_dec_ducklake_records(h, 1), C.c_uint64, np.uint64, n)) if n else []
    texts = []
    for which in range(3):
        d, o, nb = C.c_void_p(), C.c_void_p(), C.c_uint64()
        assert lib.etl_dec_ducklake_text(h, which, 1, C.byref(d), C.byref(o), C.byref(nb)) == 0
        offs = arr(o.value, C.c_uint64, np.uint64, n + 1).copy()
        data = bytes((C.c_uint8 * nb.value).from_address(d.value)) if nb.value else b""
        assert int(offs[-1]) == nb.value
        texts.append((offs, data))
    iss = abi.DuckLakeIssues()
    assert lib.etl_dec_ducklake_issues(h, C.byref(iss)) == 0
    return n, [int(k) for k in kinds], [int(r) for r in recs], texts, iss


def check(lib, h, want, what):
    n, kinds, recs, texts, iss = fetch(lib, h)
    assert n == len(want["records"]), (what, n, len(want["records"]))
    assert recs == want["records"], what
    assert kinds == want["kinds"], what
    for which in range(3):
        offs, data = texts[which]
        w = [t.encode() for t in want["texts"][which]]
        want_offs = np.zeros(n + 1, dtype=np.uint64)
        want_offs[1:] = np.cumsum([len(t) for t in w])
        for m in range(n):
            got = data[offs[m]:offs[m + 1]]
            if got != w[m]:
                raise AssertionError(f"{what}: text {which} of mutation {m}: {got[:300]!r} != {w[m][:300]!r}")
        assert np.array_equal(offs, want_offs), (what, which)
    assert (iss.first_rejected_record, iss.rejected_reason) == (want["rejected"], want["reason"]), what
    assert iss.first_empty_partial_record == want["empty"], what
    assert iss.mixed_versions == want["mixed"], what
    return n


def subs(lib, h, table, last_key=None, host=1):
    out, n = C.c_void_p(), C.c_uint64()
    key = (C.c_uint64 * 2)(*last_key) if last_key is not None else None
    rc = lib.etl_dec_ducklake_sub_batches(h, table, len(table), key, host, C.byref(out), C.byref(n))
    assert rc == 0
    if not n.value or not host:
        return n.value if not host else []
    a = (abi.DlSubBatch * n.value).from_address(out.value)
    return [(x.first_mutation, x.n_mutations, x.fingerprint) for x in a]


def check_subs(lib, h, want, what, keys=()):
    table = b"public_" + what.encode()[:20].replace(b" ", b"_")
    for key in (None,) + tuple(keys):
        got = subs(lib, h, table, key)
        exp = R.sub_batches(want, table, key)
        assert got == exp, (what, key, got[:3], exp[:3])
        for s in exp:
            assert R.batch_id(want, s).startswith("mutation:")


def names_of(planes, si, tables):
    sch = planes.schemas[si]
    cols = tables[sch.table_id]
    return [quote_ident(cols[int(i)]["name"]) for i in sch.col_index]


def run_stream(gpu, oracle_mod, tables, raw, what, first_error_ok=False, keys_of=None):
    planes, dec, st = decode(gpu, oracle_mod, tables, raw)
    if not first_error_ok:
        assert planes.first_error[0] is None, planes.first_error
    lib = abi.load()
    wants = []
    with dec.decode_input(st.view(), to_host=True) as bh:
        for si in range(len(planes.schemas)):
            names = names_of(planes, si, tables)
            want = R.expected_ducklake(planes, raw, si, names)
            rc, h = dl_emit(lib, bh, si, names)
            assert rc == 0, (what, si, rc)
            try:
                check(lib, h, want, f"{what} schema {si}")
                check_subs(lib, h, want, f"{what} {si}", keys_of(want) if keys_of else ())
                assert lib.etl_dec_ducklake_copy_fingerprint(h, b"t", 1, C.byref(C.c_uint64())) == ERR_INVALID_ARG
            finally:
                lib.etl_dec_ducklake_free(h)
            wants.append(want)
    st.close()
    dec.close()
    return planes, wants


def key_positions(want):
    """last_key in the middle of a segment, on a segment boundary, and past the end"""
    n = len(want["records"])
    if not n:
        return [(0, 0)]
    keys = [(want["commit"][n // 2], want["tx"][n // 2]), (want["commit"][-1], want["tx"][-1]), (2**64 - 1, 2**64 - 1)]
    for m in range(1, n):
        if want["seg"][m] != want["seg"][m - 1]:
            keys.append((want["commit"][m - 1], want["tx"][m - 1]))
            break
    return keys


# ------------------------------------------------------------------------------------------------ workloads
@pytest.mark.parametrize("name,scale", [("c1", 0.01), ("c2", 0.0005), ("c3", 0.001), ("c4", 0.002), ("c5", 0.0005)])
def test_workloads_match_restatement(gpu, oracle_mod, name, scale):
    w = wl.make(name, scale, n_segments=1)
    stream, _ = w.generate()
    raw = stream.tobytes()
    planes, wants = run_stream(gpu, oracle_mod, w.table_schemas(), raw, name, first_error_ok=True, keys_of=key_positions)
    assert sum(len(x["records"]) for x in wants) > 0


# ------------------------------------------------------------------------------------------------ hand-built streams
FLOATS = ["0", "-0", "1e21", "1e-7", "123456789012345680000", "5e-324", "2.2250738585072014e-308", "9007199254740993",
          "1.7976931348623157e308", "0.1", "NaN", "Infinity", "-Infinity", "1e15", "1e23", "-3.25"]


def _stream(rel_id, cols, identity, ident_names, events, name="dl"):
    w = pg.StreamWriter()
    tx = sc.Tx(w)
    tx.begin()
    w.emit(pg.relation(rel_id, "public", name, identity, sc.rel_cols(cols, ident_names)))
    for e in events:
        if e == "commit":
            tx.commit()
            tx.begin()
        else:
            w.emit(e)
    tx.commit()
    return w.bytes()


def test_hand_built_every_kind(gpu, oracle_mod):
    """every scalar type and array element kind as inserts, FULL-identity updates and deletes"""
    cols, row, n_rows = hand_built(oracle_mod)
    ev = []
    for r in range(n_rows):
        ev.append(pg.insert(95, row(r)))
        if r % 3 == 1:
            ev.append(pg.update(95, row(r + 1), old=row(r)))
        if r % 5 == 2:
            ev.append(pg.delete(95, old=row(r)))
    raw = _stream(95, cols, "f", {c["name"] for c in cols}, ev)
    planes, wants = run_stream(gpu, oracle_mod, {95: cols}, raw, "hand-built")
    assert any(k & R.MF_ARRAY for k in wants[0]["kinds"])


def test_floats_strings_json_and_quoted_names(gpu, oracle_mod):
    """float corner values (float4 and float8), strings with quotes, backslashes and UTF-8 (short and long), Json whose
    canonical text holds ' or \\, bytea, and column names that need quoting"""
    cols = [sc.col("Id", sc.INT8, 1), sc.col("f 8", 701, None, True), sc.col("f4", 700, None, True),
            sc.col('we"ird', sc.TEXT, None, True), sc.col("j", sc.JSONB, None, True), sc.col("b", 17, None, True),
            sc.col("fa", 1022, None, True)]
    strs = ["it's", "back\\slash", "é✓'\\", "x" * 70 + "'" * 5 + "\\" + "é" * 40, "", "plain"]
    docs = ['{"a":"it\'s"}', '{"b":"x\\\\y","a":[1,2]}', '"' + "q'" * 60 + '"', "[1.5e3, null, true]"]
    ev = []
    for r in range(48):
        f8, f4 = FLOATS[r % len(FLOATS)], FLOATS[(r * 5) % len(FLOATS)]
        vals = [str(r), f8, f4, strs[r % len(strs)], docs[r % len(docs)], "\\x" + ("00ff" * (r * 7 % 40)),
                "{%s,NULL,%s}" % (FLOATS[r % len(FLOATS)], FLOATS[(r + 3) % len(FLOATS)])]
        if r % 7 == 6:
            vals[3] = None
        ev.append(pg.insert(96, vals))
        if r % 4 == 1:
            ev.append(pg.update(96, vals[:3] + ["u" + strs[(r + 1) % len(strs)]] + vals[4:], old=vals))
        if r % 6 == 2:
            ev.append(pg.delete(96, old=vals))
    raw = _stream(96, cols, "f", {"Id", 'we"ird'}, ev)
    planes, wants = run_stream(gpu, oracle_mod, {96: cols}, raw, "floats strings")
    text = "".join(wants[0]["texts"][1])
    assert '"we""ird" IS NULL' in text and "E'" in "".join(wants[0]["texts"][0])


def test_identities_partials_and_rejects(gpu, oracle_mod):
    """REPLICA IDENTITY DEFAULT with key images and partial updates with and without an old image (REPLACE, key rows
    built from the partial row, a missing key column rejected, an empty partial reported); an alternative identity
    ('i' over a non-key column); a table without identity ('n') whose updates and deletes are rejected"""
    cols = [sc.col("id", sc.INT8, 1), sc.col("k2", sc.TEXT, 2), sc.col("t", sc.TEXT, None, True), sc.col("big", sc.TEXT, None, True)]
    ev = []
    for r in range(60):
        row = [str(r), f"k'{r}", "t", "b" * 300]
        ev.append(pg.insert(91, row))
        m = r % 6
        if m == 0:
            ev.append(pg.update(91, [str(r + 500), f"k'{r}", "t2", "b"], key=[str(r), f"k'{r}"]))
        elif m == 1:
            ev.append(pg.update(91, [str(r), f"k'{r}", "t3", "c"]))                       # REPLACE
        elif m == 2:
            ev.append(pg.update(91, [str(r), f"k'{r}", "t4", pg.UNCHANGED]))              # partial, key from the row
        elif m == 3:
            ev.append(pg.update(91, [str(r), f"k'{r}", None, pg.UNCHANGED], key=[str(r), f"k'{r}"]))  # partial, key image
        elif m == 4 and r > 40:
            ev.append(pg.update(91, [str(r), f"k{r}", "t5", pg.UNCHANGED, ]))
        if r % 5 == 0:
            ev.append(pg.delete(91, key=[str(r), f"k'{r}"]))
    planes, wants = run_stream(gpu, oracle_mod, {91: cols}, _stream(91, cols, "d", {"id", "k2"}, ev), "key images",
                               keys_of=key_positions)
    kinds = {k & 0x7F for k in wants[0]["kinds"]}
    assert {R.INSERT, R.UPDATE, R.UPDATE_PARTIAL, R.REPLACE, R.DELETE} <= kinds

    # alternative identity: identity over t, primary key id
    cols_i = [sc.col("id", sc.INT8, 1), sc.col("t", sc.TEXT), sc.col("u", sc.TEXT, None, True)]
    ev = [pg.insert(92, ["1", "a", "x"]), pg.update(92, ["1", "b", "y"], key=["a"]), pg.delete(92, key=["b"]),
          pg.update(92, ["2", "c", "z"]), pg.insert(92, ["3", "d", None])]
    planes, wants = run_stream(gpu, oracle_mod, {92: cols_i}, _stream(92, cols_i, "i", {"t"}, ev), "identity i")
    assert wants[0]["texts"][1][1] == "t = 'a'"

    # no identity: updates and deletes are rejected; partial key missing
    cols_n = [sc.col("id", sc.INT8, 1), sc.col("v", sc.TEXT, None, True)]
    ev = [pg.insert(93, ["1", "a"]), pg.update(93, ["1", "b"]), pg.delete(93, old=["1", "b"]), pg.insert(93, ["2", "c"])]
    planes, wants = run_stream(gpu, oracle_mod, {93: cols_n}, _stream(93, cols_n, "n", set(), ev), "no identity")
    assert wants[0]["reason"] == R.REJ_UPDATE_NO_IDENTITY
    cols_p = [sc.col("id", sc.TEXT, 1), sc.col("v", sc.TEXT, None, True)]
    ev = [pg.insert(94, ["a", "b"]), pg.update(94, [pg.UNCHANGED, "c"]), pg.update(94, ["a", pg.UNCHANGED])]
    planes, wants = run_stream(gpu, oracle_mod, {94: cols_p}, _stream(94, cols_p, "d", {"id"}, ev), "partial key",
                               first_error_ok=True)
    assert wants[0]["reason"] in (R.REJ_PARTIAL_KEY_MISSING, 0)


def test_truncate_segments_and_last_key(gpu, oracle_mod):
    """Truncate events (of this and another table) cut the runs; last_key absent, mid-run, on a run boundary and past
    the end; a second table's DML under two versions flags mixed_versions"""
    cols = [sc.col("id", sc.INT8, 1), sc.col("v", sc.TEXT, None, True)]
    w = pg.StreamWriter()
    tx = sc.Tx(w)
    tx.begin()
    w.emit(pg.relation(97, "public", "a", "d", sc.rel_cols(cols, {"id"})))
    w.emit(pg.relation(98, "public", "b", "d", sc.rel_cols(cols, {"id"})))
    k = 0
    for seg in range(6):
        for r in range(5 + 9 * seg):
            w.emit(pg.insert(97, [str(k), f"v{k}"]))
            if r % 3 == 0:
                w.emit(pg.update(97, [str(k), f"w{k}"]))
            if r % 4 == 0:
                w.emit(pg.delete(97, key=[str(k)]))
            k += 1
            if r % 7 == 3:
                tx.commit()
                tx.begin()
        w.emit(pg.truncate([98] if seg % 2 else [97]))
        if seg == 3:                                        # table b changes version inside a run
            w.emit(pg.insert(98, ["1", "x"]))
            w.emit(pg.relation(98, "public", "b", "d", sc.rel_cols(cols + [sc.col("z", sc.INT4, None, True)], {"id"})))
            w.emit(pg.insert(98, ["2", "y", "3"]))
    tx.commit()
    raw = w.bytes()
    tables = {97: cols, 98: cols + [sc.col("z", sc.INT4, None, True)]}
    planes, wants = run_stream(gpu, oracle_mod, tables, raw, "truncates", keys_of=key_positions)
    assert len(set(wants[0]["seg"])) == 6
    assert any(x["mixed"] for x in wants[1:])


# ------------------------------------------------------------------------------------------------ COPY batches
def copy_want(oracle_mod, oids, rows, names, pk):
    cells = []
    for row in rows:
        e, _, cs, text, heap = oracle_mod.parse_copy_row(oids, row)
        if e:
            break
        cells.append([(t, decode_cell(t, v, a, text, heap)) for t, v, a in cs])
    return R.expected_copy_ducklake(cells, names, pk)


@pytest.mark.parametrize("idx", range(len(REF_ROWS)))
def test_copy_reference_vectors(gpu, oracle_mod, idx):
    oids, row = REF_ROWS[idx]
    lib = abi.load()
    dec = gpu.Decoder(0)
    cols = cols_of(oids)
    dec.put_table_schema(7, cols)
    names = [c["name"] for c in cols]
    with copy_batch(gpu, dec, 7, [row]) as bh:
        rc, h = dl_emit(lib, bh, 0, names)
        assert rc == 0
        want = copy_want(oracle_mod, oids, [row], names, [c["pk"] is not None for c in cols])
        check(lib, h, want, f"vector {idx}")
        fp = C.c_uint64()
        assert lib.etl_dec_ducklake_copy_fingerprint(h, b"public_t", 8, C.byref(fp)) == 0
        assert fp.value == R.copy_fingerprint(want, b"public_t")
        assert lib.etl_dec_ducklake_sub_batches(h, b"t", 1, None, 1, C.byref(C.c_void_p()), C.byref(C.c_uint64())) == ERR_INVALID_ARG
        lib.etl_dec_ducklake_free(h)
        assert dl_emit(lib, bh, 1, names)[0] == ERR_INVALID_ARG
    dec.close()


@pytest.mark.parametrize("n,bad_at", [(5000, 3777), (200000, None)])
def test_copy_synthetic_tables(gpu, oracle_mod, n, bad_at):
    oids, rows = synth_rows(n, 4321 + n, bad_at)
    lib = abi.load()
    dec = gpu.Decoder(0)
    cols = cols_of(oids)
    dec.put_table_schema(7, cols)
    names = [c["name"] for c in cols]
    with copy_batch(gpu, dec, 7, rows) as bh:
        want = copy_want(oracle_mod, oids, rows, names, [c["pk"] is not None for c in cols])
        assert len(want["records"]) == (bad_at if bad_at is not None else n)
        for to_host in (1, 0):
            rc, h = dl_emit(lib, bh, 0, names, to_host)
            assert rc == 0
            fp = C.c_uint64()
            if to_host:
                check(lib, h, want, f"copy {n}")
                assert lib.etl_dec_ducklake_copy_fingerprint(h, b"public_t", 8, C.byref(fp)) == 0
                assert fp.value == R.copy_fingerprint(want, b"public_t")
            else:
                assert lib.etl_dec_ducklake_kinds(h, 1) is None and lib.etl_dec_ducklake_kinds(h, 0)
                assert lib.etl_dec_ducklake_copy_fingerprint(h, b"public_t", 8, C.byref(fp)) == ERR_INVALID_ARG
            lib.etl_dec_ducklake_free(h)
    dec.close()


# ------------------------------------------------------------------------------------------------ errors, arguments, lifetime
def test_mid_batch_decode_error_and_arguments(gpu, oracle_mod):
    cols = [sc.col("id", sc.INT8, 1), sc.col("n", sc.NUMERIC, None, True), sc.col("j", sc.JSONB, None, True), sc.col("a", 1231, None, True)]
    ev = [pg.insert(99, [str(r), "%d.5" % r if r != 23 else "1.2.3", '{"r":%d,"a":[%d]}' % (r, r), "{%d,1.50}" % r]) for r in range(40)]
    raw = _stream(99, cols, "d", {"id"}, ev)
    tables = {99: cols}
    planes, dec, st = decode(gpu, oracle_mod, tables, raw)
    assert planes.first_error[0] is not None
    lib = abi.load()
    names = names_of(planes, 0, tables)
    with dec.decode_input(st.view(), to_host=True) as bh:
        want = R.expected_ducklake(planes, raw, 0, names)
        rc, h = dl_emit(lib, bh, 0, names)
        assert rc == 0
        assert check(lib, h, want, "mid-batch error") == 23
        lib.etl_dec_ducklake_free(h)
        assert dl_emit(lib, bh, len(planes.schemas), names)[0] == ERR_INVALID_ARG
        assert dl_emit(lib, bh, 0, names[:-1])[0] == ERR_INVALID_ARG
        assert lib.etl_dec_ducklake_emit(bh._h, 0, None, len(names), 1, C.byref(C.c_void_p())) == ERR_INVALID_ARG
        a = (C.c_char_p * len(names))(*[n.encode() for n in names])
        assert lib.etl_dec_ducklake_emit(bh._h, 0, a, len(names), 1, None) == ERR_INVALID_ARG
        rc, h = dl_emit(lib, bh, 0, names, to_host=0)
        assert rc == 0
        d, o, nb = C.c_void_p(), C.c_void_p(), C.c_uint64()
        assert lib.etl_dec_ducklake_text(h, 3, 0, C.byref(d), C.byref(o), C.byref(nb)) == ERR_INVALID_ARG
        assert lib.etl_dec_ducklake_text(h, 0, 1, C.byref(d), C.byref(o), C.byref(nb)) == ERR_INVALID_ARG
        assert lib.etl_dec_ducklake_text(h, 0, 0, C.byref(d), C.byref(o), C.byref(nb)) == 0 and d.value
        assert subs(lib, h, b"public_t", None, host=0) == len(R.sub_batches(want, b"public_t"))
        lib.etl_dec_ducklake_free(h)
    st.close()
    dec.close()


def test_emit_free_cycles_keep_memory_stable(gpu, oracle_mod):
    cols, row, n_rows = hand_built(oracle_mod)
    ev = [pg.insert(95, row(r)) for r in range(n_rows)]
    raw = _stream(95, cols, "f", {c["name"] for c in cols}, ev)
    tables = {95: cols}
    planes, dec, st = decode(gpu, oracle_mod, tables, raw)
    lib = abi.load()
    names = names_of(planes, 0, tables)
    free, total = C.c_uint64(), C.c_uint64()
    with dec.decode_input(st.view(), to_host=True) as bh:
        for i in range(100):
            rc, h = dl_emit(lib, bh, 0, names, to_host=1 - i % 2)
            assert rc == 0
            subs(lib, h, b"public_t", None, host=i % 2)
            lib.etl_dec_ducklake_free(h)
            assert lib.etl_dec_mem_info(dec._ctx, C.byref(free), C.byref(total)) == 0
            if i == 1:
                base = free.value
        assert abs(free.value - base) <= 4 << 20, (free.value, base)
    st.close()
    dec.close()
