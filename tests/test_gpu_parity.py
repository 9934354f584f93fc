"""GPU parity: the CUDA decode path (through the C ABI) vs the CPU oracle, bit-exact.

Runs on an H100 (`pytest -m gpu`).  Nothing here reads the reference checkout.
"""
import numpy as np
import pytest

import scenarios as sc
from canon import assert_planes_equal, planes_to_events
from etl_b200 import pgoutput as pg
from etl_b200 import workloads as wl

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def gpu():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from etl_b200 import decoder
    return decoder


def both(gpu, oracle_mod, tables, stream, carry=None, stride=2048):
    dec = gpu.Decoder(0)
    orc = oracle_mod.Oracle()
    for tid, cols in tables.items():
        dec.put_table_schema(tid, cols)
        orc.put_table_schema(tid, cols)
    got = dec.decode(stream, carry, anchor_stride=stride)
    want = orc.decode(stream, carry)
    dec.close()
    return got, want


def dml(events):
    return [{k: e[k] for k in ("kind", "row", "old") if k in e} for e in events if e["kind"] in ("insert", "update", "delete")]


@pytest.mark.parametrize("name,tables,w,expected", sc.reference_update_delete_scenarios() + sc.tuple_level_scenarios(),
                         ids=lambda x: x if isinstance(x, str) else None)
def test_reference_event_vectors_on_gpu(gpu, oracle_mod, name, tables, w, expected):
    stream = w.bytes()
    got, want = both(gpu, oracle_mod, tables, stream)
    assert_planes_equal(got, want, stream)
    if not (isinstance(expected, tuple) and expected[0] == "error"):
        assert dml(planes_to_events(got, stream)) == expected
    else:
        assert got.first_error[2] == expected[1]


@pytest.mark.parametrize("name,tables,w,expected", sc.error_scenarios(), ids=lambda x: x if isinstance(x, str) else None)
def test_error_scenarios_on_gpu(gpu, oracle_mod, name, tables, w, expected):
    stream = w.bytes()
    got, want = both(gpu, oracle_mod, tables, stream)
    assert (got.first_error[0], got.first_error[2]) == expected
    assert_planes_equal(got, want, stream)


@pytest.mark.parametrize("name,scale", [("c1", 1.0), ("c2", 0.05), ("c3", 0.01), ("c4", 0.004), ("c5", 0.003)])
@pytest.mark.parametrize("stride", [2048, 512, 16384])
def test_workload_parity(gpu, oracle_mod, name, scale, stride):
    w = wl.make(name, scale)
    stream, stats = w.generate()
    got, want = both(gpu, oracle_mod, w.table_schemas(), stream, stride=stride)
    assert want.first_error[0] is None
    assert got.n_records == stats["frames"]
    assert_planes_equal(got, want, stream.tobytes(), check_heap_contents=(name != "c3" or stride == 2048))


def test_mid_transaction_carry(gpu, oracle_mod):
    """A batch that starts inside a transaction (carry-in) and ends inside another (carry-out)."""
    w = wl.make("c2", 0.01, n_segments=1)
    stream, _ = w.generate()
    o = oracle_mod.Oracle()
    for tid, cols in w.table_schemas().items():
        o.put_table_schema(tid, cols)
    full = o.decode(stream)
    # cut at a record boundary in the middle of a transaction
    cut_rec = next(i for i in range(full.n_records // 2, full.n_records) if chr(full.rec_kind[i]) in "IUD" and chr(full.rec_kind[i + 1]) in "IUD")
    cut = int(full.rec_off[cut_rec + 1])
    a, b = stream[:cut], stream[cut:]
    dec = gpu.Decoder(0)
    orc = oracle_mod.Oracle()
    for tid, cols in w.table_schemas().items():
        dec.put_table_schema(tid, cols)
        orc.put_table_schema(tid, cols)
    g1, w1 = dec.decode(a), orc.decode(a)
    assert_planes_equal(g1, w1, a.tobytes())
    assert g1.carry_out[0] == 1
    g2, w2 = dec.decode(b, g1.carry_out), orc.decode(b, w1.carry_out)
    assert_planes_equal(g2, w2, b.tobytes())
    assert int(g2.rec_tx_ordinal[0]) == int(full.rec_tx_ordinal[cut_rec + 1])
    assert int(g2.rec_commit_lsn[0]) == int(full.rec_commit_lsn[cut_rec + 1])
    dec.close()


def test_error_in_large_stream_valid_prefix(gpu, oracle_mod):
    """first_error = the earliest failing record; everything before it is bit-exact."""
    w = wl.make("c2", 0.02, n_segments=2)
    stream, _ = w.generate()
    o = oracle_mod.Oracle()
    for tid, cols in w.table_schemas().items():
        o.put_table_schema(tid, cols)
    full = o.decode(stream)
    s = bytearray(stream.tobytes())
    # corrupt an int4 cell ("x" is not a digit) in two different records; the earlier one must win
    victims = [i for i in range(full.n_records) if chr(full.rec_kind[i]) == "I"]
    for rec in (victims[len(victims) // 2], victims[len(victims) // 3]):
        off = int(full.rec_off[rec])
        # first tuple cell of an insert: 'd' len 'w' hdr(24) 'I' rel(4) 'N' ncols(2) 't' len(4) value
        assert s[off + 38:off + 39] == b"t"
        s[off + 43] = ord("x")
    s = bytes(s)
    got, want = both(gpu, oracle_mod, w.table_schemas(), s)
    assert want.first_error[0] == victims[len(victims) // 3] and want.first_error[2] == 2
    assert_planes_equal(got, want, s)


def test_big_cells_and_oversize_frames(gpu, oracle_mod):
    """TOAST-sized text: cooperative UTF-8 validation, frames larger than the shared-memory window,
    and an invalid byte deep inside a 100 KiB value."""
    cols = [sc.col("id", sc.INT8, 1), sc.col("doc", sc.TEXT, None, True), sc.col("n", sc.INT4, None, True)]
    rel = pg.relation(90, "public", "docs", "f", sc.rel_cols(cols, set()))
    rng = np.random.default_rng(7)

    def text(n, nonascii=True):
        b = bytearray(rng.integers(97, 123, size=n, dtype=np.uint8).tobytes())
        if nonascii:
            for pos in range(3, n - 8, 97):
                b[pos:pos + 4] = "🤔".encode()
        return bytes(b)

    w = pg.StreamWriter()
    tx = sc.Tx(w)
    tx.begin()
    w.emit(rel)
    sizes = [511, 512, 513, 2000, 8191, 33000, 40960, 70000, 150000]
    for i, n in enumerate(sizes):
        w.emit(pg.insert(90, [str(i), text(n), str(n)]))
        w.emit(pg.update(90, [str(i), pg.UNCHANGED, "5"], old=[str(i), text(n), "4"]))
    tx.commit()
    stream = w.bytes()
    got, want = both(gpu, oracle_mod, {90: cols}, stream)
    assert want.first_error[0] is None
    assert_planes_equal(got, want, stream)
    # now poison one byte in the middle of the 70000-byte value
    bad = bytearray(stream)
    rec = 2 + 2 * sizes.index(70000)
    pos = int(want.rec_off[rec]) + 50000
    bad[pos] = 0xFF
    bad = bytes(bad)
    got, want = both(gpu, oracle_mod, {90: cols}, bad)
    assert want.first_error[0] == rec and want.first_error[2] == 1
    assert_planes_equal(got, want, bad)


def _two_phase(gpu, tables, raw, cuts):
    """The multi-GPU protocol on one device: every range runs decode_begin (index + scan → seam summary), the
    summaries are folded exactly as after an all-gather, decode_finish gets the carry and the global record base."""
    from etl_b200 import sharding
    from etl_b200.decoder import Stager
    dec = gpu.Decoder(0)
    for tid, cols in tables.items():
        dec.put_table_schema(tid, cols)
    parts, state, base = [], (0, 0, 0), 0
    for k in range(len(cuts) - 1):
        shard = raw[cuts[k]:cuts[k + 1]]
        st = Stager(len(shard), 2048)
        st.append_framed(shard)
        seam = dec.decode_begin(st.view(), to_host=True)
        words = sharding.seam_to_words(seam)
        with dec.decode_finish(state, base) as bh:
            parts.append(bh.to_host())
        state = sharding.fold_state(state, words)
        base += int(words[0])
        st.close()
    dec.close()
    return parts, base


def test_two_phase_shards_with_seam_fold(gpu, oracle_mod):
    """Cuts are in the middle of transactions; the stitched result must equal the oracle's decode of the whole
    stream on EVERY plane."""
    from shard_util import mid_tx_cuts, stitch
    w = wl.make("c2", 0.02, n_segments=1)
    stream, _ = w.generate()
    raw = stream.tobytes()
    orc = oracle_mod.Oracle()
    for tid, cols in w.table_schemas().items():
        orc.put_table_schema(tid, cols)
    full = orc.decode(raw)
    cuts = mid_tx_cuts(full, 3) + [len(raw)]
    parts, base = _two_phase(gpu, w.table_schemas(), raw, cuts)
    assert base == full.n_records
    assert all(p.first_error[0] is None for p in parts)
    assert_planes_equal(stitch(parts, cuts), full, raw)


def test_two_phase_error_in_later_shard_reports_global_index(gpu, oracle_mod):
    """A data error in the third range carries its GLOBAL record index (record_index_base > 0 in report_error and
    k_long_cells), and is the index the oracle reports for the whole stream."""
    from shard_util import mid_tx_cuts
    w = wl.make("c2", 0.02, n_segments=1)
    stream, _ = w.generate()
    orc = oracle_mod.Oracle()
    for tid, cols in w.table_schemas().items():
        orc.put_table_schema(tid, cols)
    full = orc.decode(stream.tobytes())
    cuts = mid_tx_cuts(full, 3)
    s = bytearray(stream.tobytes())
    victim = next(i for i in range(full.n_records * 5 // 6, full.n_records) if chr(full.rec_kind[i]) == "I")
    off = int(full.rec_off[victim])
    assert off > cuts[2] and s[off + 38:off + 39] == b"t"
    s[off + 43] = ord("x")                              # first cell (int4) of an insert: not a digit any more
    raw = bytes(s)
    want = orc.decode(raw)
    assert want.first_error[0] == victim
    parts, _ = _two_phase(gpu, w.table_schemas(), raw, cuts + [len(raw)])
    assert parts[0].first_error[0] is None and parts[1].first_error[0] is None
    assert parts[2].first_error == want.first_error


FLOAT_CASES = ["0", "-0", "1", "3.15", "-2.818", "inf", "-Infinity", "NaN", "-nan", "3.4028235e38", "-3.4028235e38",
               "1.7976931348623157e308", "1e999", "1e-999", "4.9406564584124654e-324", "2.4703282292062327e-324",
               "2.4703282292062328e-324", "2.2250738585072011e-308", "2.2250738585072014e-308", "9007199254740993",
               "9007199254740992.99999999999999999", "16777217", "16777216.000000000000000000000001",
               "1.00000017881393432617187499", "1.00000017881393432617187501", "0.1", "0.30000000000000004", "1e23",
               "8.41e21", "123456789012345678901234567890", "0.000000000000000000000000000000000000000000001",
               "1.", ".5", "+1e3", "1E-2", "5e-324", "1e308", "1.8e308", "7.038531e-26", "1.17549435e-38",
               "1.401298464324817e-45", "7.006492321624085e-46", "7.006492321624086e-46",
               "340282356779733661637539395458142568448", "179769313486231580793728971405303415079934132710037826936173778980444968292764750946649017977587207096330286416692887910946555547851940402630657488671505820681908902000708383676273854845817711531764475730270069855571366959622842914819860834936475292719074168444365510704342711559699508093042880177904174497792",
               "", ".", "e5", "1e", "1e+", " 1", "1 ", "+", "-", "1_0", "0x1p3", "infinit", "nan(1)", "1.2.3"]


def test_float_parity(gpu, oracle_mod):
    """float4 / float8 (text.rs:61-68): every value alone in its own stream so that invalid spellings
    (→ first_error) and valid ones are both compared with the oracle (glibc strtod/strtof, correctly rounded)."""
    cols = [sc.col("id", sc.INT8, 1), sc.col("f8", sc.FLOAT8, None, True), sc.col("f4", 700, None, True)]
    rel = pg.relation(91, "public", "floats", "d", sc.rel_cols(cols, {"id"}))
    rng = np.random.default_rng(11)
    cases = list(FLOAT_CASES)
    for _ in range(300):
        mant = "".join(str(d) for d in rng.integers(0, 10, size=int(rng.integers(1, 30))))
        cases.append(f"{mant[:1]}.{mant[1:]}e{int(rng.integers(-330, 320))}")
        cases.append(repr(float(rng.standard_normal() * 10.0 ** int(rng.integers(-30, 30)))))
    # valid values: one big stream
    w = pg.StreamWriter()
    tx = sc.Tx(w)
    tx.begin()
    w.emit(rel)
    valid = [c for c in cases if oracle_mod.parse_cell(701, c.encode())[0] == 0]
    for i, c in enumerate(valid):
        w.emit(pg.insert(91, [str(i), c, c]))
    tx.commit()
    stream = w.bytes()
    got, want = both(gpu, oracle_mod, {91: cols}, stream)
    assert want.first_error[0] is None and len(valid) > 600
    assert_planes_equal(got, want, stream)
    for c in [c for c in cases if c not in valid]:
        w = pg.StreamWriter()
        tx = sc.Tx(w)
        tx.begin()
        w.emit(rel)
        w.emit(pg.insert(91, ["1", c, None]))
        tx.commit()
        got, want = both(gpu, oracle_mod, {91: cols}, w.bytes())
        assert want.first_error[2] == 3, c
        assert got.first_error == want.first_error, c


# ---------------------------------------------------------------------------------------------
# arrays (SURVEY §8a row 13; text.rs:69-140 element dispatch, :184-249 the split)
# ---------------------------------------------------------------------------------------------
ARRAY_COLS = [  # (array type oid, valid spellings, invalid spellings)
    (1007, ["{}", "{1,2,3}", "{NULL,5,null}", '{"7","-8"}', "{2147483647,-2147483648}"], ["{1,x}", "{2147483648}", "1,2", "{", "{1,2", "{1,,2}"]),
    (1016, ["{9223372036854775807}", "{+5}"], ["{9223372036854775808}"]),
    (1005, ["{1,-32768}"], ["{40000}"]),
    (1000, ["{t,f,NULL}"], ["{true}"]),
    (1009, ['{a,b c,"d,e","f\\"g",NULL,"NULL","",\\x}', '{"multi\\\\back","é✓"}', "{ a , b }"], []),
    (1022, ["{1.5,-2e10,NaN,inf,NULL}"], ["{1.5,abc}"]),
    (1021, ["{0.1,3.4028235e38}"], ["{}x"]),
    (1231, ["{1.50,NaN,-0.0001,123456789012345678901234567890.123456789,NULL}"], ["{1.2.3}"]),
    (1182, ["{2024-01-02,0001-01-01}"], ["{2024-13-01}"]),
    (1183, ["{12:34:56.789,00:00:00}"], ["{25:00:00}"]),
    (1115, ['{"2024-01-02 03:04:05.678","2000-02-29 23:59:59"}'], ['{"2024-01-02"}']),
    (1185, ['{"2024-01-02 03:04:05+00","2024-06-01 12:00:00.5-07"}', '{"2024-01-02 03:04:05+05:30"}',
            '{"2024-01-02 03:04:05+05:30","2024-01-02 03:04:05+00"}'], ['{"2024-01-02 03:04:05"}', '{"2024-01-02 03:04:05+5"}']),
    (2951, ["{a0eebc99-9c0b-4ef8-bb6d-6bb9bd380a11,NULL}"], ["{zz}"]),
    (199, ['{"{\\"a\\": [1, 2]}","null",NULL}'], ['{"{bad"}']),
    (3807, ['{"[1,2,3]"}'], ['{"[1,"}']),
    (1001, ['{"\\\\x0102ff",NULL}'], ['{"\\\\x0g"}', "{abc}"]),
    (1028, ["{1,4294967295}"], ["{-1}"]),
]


def test_array_parity(gpu, oracle_mod):
    """Every array element kind the reference decodes: valid spellings together in one stream, then each
    invalid spelling alone (first_error compared).  Heap placement is unspecified; contents are compared."""
    usable = [(oid, v, bad) for oid, v, bad in ARRAY_COLS if oracle_mod.kind_for_oid(oid) & 0x20]
    assert len(usable) >= 12, [hex(oracle_mod.kind_for_oid(o)) for o, _, _ in ARRAY_COLS]
    cols = [sc.col("id", sc.INT8, 1)] + [sc.col(f"a{oid}", oid, None, True) for oid, _, _ in usable]
    rel = pg.relation(92, "public", "arrays", "d", sc.rel_cols(cols, {"id"}))
    w = pg.StreamWriter()
    tx = sc.Tx(w)
    tx.begin()
    w.emit(rel)
    nrow = max(len(v) for _, v, _ in usable)
    for r in range(nrow * 40):   # enough rows to overflow the first heap guess? no: to exercise many warps
        w.emit(pg.insert(92, [str(r)] + [v[(r + j) % len(v)] for j, (_, v, _) in enumerate(usable)]))
    tx.commit()
    stream = w.bytes()
    got, want = both(gpu, oracle_mod, {92: cols}, stream)
    assert want.first_error[0] is None, want.first_error
    assert_planes_equal(got, want, stream)
    for j, (oid, _, bads) in enumerate(usable):
        for bad in bads:
            w = pg.StreamWriter()
            tx = sc.Tx(w)
            tx.begin()
            w.emit(rel)
            vals = [None] * len(usable)
            vals[j] = bad
            w.emit(pg.insert(92, ["1"] + vals))
            tx.commit()
            got, want = both(gpu, oracle_mod, {92: cols}, w.bytes())
            assert want.first_error[0] is not None, (oid, bad)
            assert got.first_error == want.first_error, (oid, bad, got.first_error, want.first_error)


def test_array_heap_retry(gpu, oracle_mod):
    """Arrays of many empty elements need far more heap than the first reservation (44 B per element):
    the decode retries with a larger heap instead of failing or truncating."""
    cols = [sc.col("id", sc.INT8, 1), sc.col("a", 1009, None, True)]
    rel = pg.relation(93, "public", "wide", "d", sc.rel_cols(cols, {"id"}))
    w = pg.StreamWriter()
    tx = sc.Tx(w)
    tx.begin()
    w.emit(rel)
    for r in range(64):
        w.emit(pg.insert(93, [str(r), "{" + "," * 3000 + "}"]))
    tx.commit()
    stream = w.bytes()
    got, want = both(gpu, oracle_mod, {93: cols}, stream)
    assert want.first_error[0] is None
    assert_planes_equal(got, want, stream)


def test_long_cell_utf8_boundaries(gpu, oracle_mod):
    """Long text takes its interior UTF-8 verdict from the structure-blind line bitmap and its head / tail
    from direct checks: poison bytes (and split multi-byte sequences) at every kind of position — first
    bytes of the cell, around the first and last 128-byte line boundary, the last bytes — and valid
    multi-byte sequences that straddle line boundaries.  Verdicts must match the oracle byte for byte."""
    cols = [sc.col("id", sc.INT8, 1), sc.col("doc", sc.TEXT, None, True)]
    rel = pg.relation(94, "public", "docs2", "d", sc.rel_cols(cols, {"id"}))
    rng = np.random.default_rng(5)
    n = 3000

    def build(payload: bytes) -> bytes:
        w = pg.StreamWriter()
        tx = sc.Tx(w)
        tx.begin()
        w.emit(rel)
        w.emit(pg.insert(94, ["1", "pad" * 7]))
        w.emit(_raw_text_insert(94, b"2", payload))
        tx.commit()
        return w.bytes()

    base = bytearray(rng.integers(97, 123, size=n, dtype=np.uint8).tobytes())
    clean = build(bytes(base))
    got, want = both(gpu, oracle_mod, {94: cols}, clean)
    assert want.first_error[0] is None
    assert_planes_equal(got, want, clean)
    cell_off = clean.index(bytes(base))            # absolute stream offset of the value
    l0 = (-(cell_off + 3)) % 128 + 3               # cell-relative offset of the first interior line
    last_line = (cell_off + n) // 128 * 128 - cell_off
    spots = sorted({0, 1, 2, 3, l0 - 4, l0 - 1, l0, l0 + 1, l0 + 127, l0 + 128, 1500, last_line - 1, last_line, last_line + 1, n - 4, n - 2, n - 1})
    emoji = "🤔".encode()
    for p in spots:
        for kind in ("ff", "cont", "lead", "emoji"):
            b = bytearray(base)
            if kind == "ff":
                b[p] = 0xFF
            elif kind == "cont":
                b[p] = 0x80                          # continuation byte without a lead
            elif kind == "lead":
                b[p] = 0xE2                          # lead byte followed by ASCII (or by the end of the cell)
            else:
                if p + 4 > n:
                    continue
                b[p:p + 4] = emoji                   # valid 4-byte sequence, possibly straddling a line boundary
            s = build(bytes(b))
            got, want = both(gpu, oracle_mod, {94: cols}, s)
            assert got.first_error == want.first_error, (p, kind, got.first_error, want.first_error)
            assert (want.first_error[0] is None) == (kind == "emoji"), (p, kind)


def test_frame_length_hint_is_only_a_hint(gpu, oracle_mod):
    """etl_dec_input.max_frame_len lets the decoder leave out the passes that exist for long values.  Three cases on a
    stream WITH long values (C5: TOASTed text, one value poisoned with an invalid byte deep inside): the stager's own
    (correct) hint, no hint, and a hint that wrongly promises short frames — the planes and the error must not change."""
    w = wl.make("c5", 0.003, n_segments=1)
    stream, _ = w.generate()
    raw = bytearray(stream.tobytes())
    tables = w.table_schemas()
    orc0 = oracle_mod.Oracle()
    for tid, cols in tables.items():
        orc0.put_table_schema(tid, cols)
    clean = orc0.decode(bytes(raw))
    longs = np.flatnonzero((np.asarray(clean.cell_tag) == 2) & (np.asarray(clean.cell_aux) > 8192))   # String cells of TOAST size
    assert len(longs) > 4
    victim = int(longs[len(longs) // 2])
    for poison in (False, True):
        data = bytes(raw)
        if poison:
            b = bytearray(data)
            b[int(clean.cell_val[victim]) + int(clean.cell_aux[victim]) // 2] = 0xFF     # deep inside the value: a dead segment
            data = bytes(b)
        orc = oracle_mod.Oracle()
        for tid, cols in tables.items():
            orc.put_table_schema(tid, cols)
        want = orc.decode(data)
        assert (want.first_error[0] is not None) == poison
        for hint in (None, 0, 64):
            dec = gpu.Decoder(0)
            for tid, cols in tables.items():
                dec.put_table_schema(tid, cols)
            got = dec.decode(data, max_frame_len=hint)
            dec.close()
            assert got.first_error == want.first_error, (poison, hint, got.first_error, want.first_error)
            if not poison:
                assert_planes_equal(got, want, data)


def _raw_text_insert(rel_id: int, key: bytes, payload: bytes) -> bytes:
    """Insert message whose second column carries arbitrary bytes (pg.insert encodes str as UTF-8)."""
    import struct
    body = b"I" + struct.pack(">I", rel_id) + b"N" + struct.pack(">H", 2)
    body += b"t" + struct.pack(">I", len(key)) + key + b"t" + struct.pack(">I", len(payload)) + payload
    return body


# ---------------------------------------------------------------------------------------------
# seeded fuzz over every scalar decode class: canonical spellings and mutations of them
# ---------------------------------------------------------------------------------------------
FUZZ_KINDS = [  # (type oid, canonical spellings, alphabet used for mutations)
    (21, ["0", "-32768", "32767", "+7", "12"], "0123456789+- _x"),
    (23, ["0", "-2147483648", "2147483647", "+15", "000123"], "0123456789+- _.e"),
    (20, ["0", "-9223372036854775808", "9223372036854775807", "18446744073709551615", "42"], "0123456789+- "),
    (26, ["0", "4294967295", "4294967296", "-1", "16384"], "0123456789+-"),
    (16, ["t", "f", "true", "T", ""], "tfTF01 "),
    (1700, ["0", "-0.00", "123.456", "NaN", "Infinity", "-Infinity", "1e10", "0.000000001", "99999999999999999999.0001", "1_000", ".5", "5.", "+1.5E-3"],
     "0123456789.+-eE_NaInfity "),
    (1082, ["2024-02-29", "0001-01-01", "9999-12-31", "2023-02-29", "2024-1-5", " 2024-01-05", "2024-01-05 ", "+2024-01-05", "10000-01-01", "-0001-01-01"],
     "0123456789-+ /"),
    (1083, ["00:00:00", "23:59:59.999999", "12:34:56.1", "24:00:00", "12:34", "12:34:60", "1:2:3", "12:34:56.1234567891"], "0123456789:. "),
    (1114, ["2024-02-29 12:34:56", "2024-02-29 12:34:56.789", "2024-02-29T12:34:56", "2024-02-29 24:00:00", "2024-02-30 00:00:00",
            "1-1-1 1:1:1", "2024-02-29  12:34:56", "2024-02-29 12:34:56.", "2024-02-29 12:34:60"], "0123456789-:. T"),
    (1184, ["2024-02-29 12:34:56+00", "2024-02-29 12:34:56.789-07", "2024-02-29 12:34:56+05:30", "2024-02-29 12:34:56+0530", "2024-02-29 12:34:56Z",
            "2024-02-29 12:34:56 +00", "2024-02-29 12:34:56+24", "2024-02-29 12:34:56+5", "2024-02-29 12:34:56+05:3", "2024-02-29 12:34:56.123456789+00:00:00"],
     "0123456789-:. +Zz"),
    (2950, ["a0eebc99-9c0b-4ef8-bb6d-6bb9bd380a11", "A0EEBC99-9C0B-4EF8-BB6D-6BB9BD380A11", "a0eebc999c0b4ef8bb6d6bb9bd380a11",
            "{a0eebc99-9c0b-4ef8-bb6d-6bb9bd380a11}", "urn:uuid:a0eebc99-9c0b-4ef8-bb6d-6bb9bd380a11", "a0eebc99-9c0b-4ef8-bb6d-6bb9bd380a1"],
     "0123456789abcdefABCDEFg-{}"),
    (17, ["\\x", "\\x00ff", "\\xDEADbeef", "\\x0", "abc", "\\\\000", "\\x+f", ""], "\\x0123456789abcdefABCDEFg+ "),
    (3802, ['{"a": 1}', "[1, 2.5, -3e2]", '"s"', "null", " true ", '{"a": {"b": [null, false]}}', '"\\u00e9"', '"\\ud83d\\ude00"', "01", "{", '{"a" 1}'],
     '{}[]":, 0123456789.-+eEtruefalsn\\ud8'),
    (25, ["", "plain", "with space", "unicode é ✓ 🤔", "x" * 300], "abc é✓"),
    (701, ["0", "-1.5", "1e308", "1e309", "NaN", "-inf", "4.9e-324", "0.1", "1.7976931348623157e308", "2.2250738585072011e-308"], "0123456789.+-eEnaif"),
    (700, ["0", "-1.5", "3.4028235e38", "3.4028236e38", "1e-45", "0.1", "16777217"], "0123456789.+-eE"),
]


@pytest.mark.parametrize("oid", [k[0] for k in FUZZ_KINDS])
def test_scalar_fuzz_parity(gpu, oracle_mod, oid):
    """Per decode class: the canonical spellings above and ~300 seeded mutations of them (insert / delete /
    replace from a class-specific alphabet).  Values the oracle accepts go into one stream (every typed value
    compared); values it rejects are decoded one per stream (error kind and position compared)."""
    _, seeds, alphabet = next(k for k in FUZZ_KINDS if k[0] == oid)
    rng = np.random.default_rng(oid)
    cases = list(seeds)
    for _ in range(300):
        s = list(seeds[int(rng.integers(0, len(seeds)))])
        for _ in range(int(rng.integers(1, 3))):
            op = int(rng.integers(0, 3))
            p = int(rng.integers(0, len(s) + 1))
            ch = alphabet[int(rng.integers(0, len(alphabet)))]
            if op == 0:
                s.insert(p, ch)
            elif op == 1 and s:
                del s[min(p, len(s) - 1)]
            elif s:
                s[min(p, len(s) - 1)] = ch
        cases.append("".join(s))
    cases = list(dict.fromkeys(cases))
    cols = [sc.col("id", sc.INT8, 1), sc.col("v", oid, None, True)]
    rel = pg.relation(95, "public", "fuzz", "d", sc.rel_cols(cols, {"id"}))
    valid = [c for c in cases if oracle_mod.parse_cell(oid, c.encode())[0] == 0]
    invalid = [c for c in cases if c not in valid]
    assert valid, oid
    w = pg.StreamWriter()
    tx = sc.Tx(w)
    tx.begin()
    w.emit(rel)
    for i, c in enumerate(valid):
        w.emit(pg.insert(95, [str(i), c]))
    tx.commit()
    stream = w.bytes()
    got, want = both(gpu, oracle_mod, {95: cols}, stream)
    assert want.first_error[0] is None
    assert_planes_equal(got, want, stream)
    for c in invalid[:120]:
        w = pg.StreamWriter()
        tx = sc.Tx(w)
        tx.begin()
        w.emit(rel)
        w.emit(pg.insert(95, ["1", c]))
        tx.commit()
        got, want = both(gpu, oracle_mod, {95: cols}, w.bytes())
        assert want.first_error[0] is not None, (oid, c)
        assert got.first_error == want.first_error, (oid, c, got.first_error, want.first_error)
