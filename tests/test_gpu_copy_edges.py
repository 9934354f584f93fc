"""COPY-text rows on the device (etl_dec_copy_decode: k_copy_rows + k_heavy) at the edges where the kernels change
strategy, each compared with the oracle's restatement of parse_table_row_from_postgres_copy_bytes:

* heap sizing: short escaped fields (an 8-byte heap copy each), escaped heavy values parsed by k_heavy from their heap
  copy, and uuid fields the light pass declines (a slot in each kernel) — plus the replication path's declined uuids;
* the staging window (ETL_ROWS_WIN bytes from the row start rounded down to 16): separators, escapes, NULL markers
  and 4-byte UTF-8 at every offset around the first and second window end, for every row start modulo 16;
* fields longer than a window in every decode class (read from global memory, or by k_heavy without staging);
* lanes of one warp in different states: batch sizes around 32 and 128, long rows among short ones, light and heavy
  classes alternating, rows with too few and too many fields;
* column counts around the 256 column kinds k_copy_rows keeps in shared memory, and zero columns;
* which error is reported first: UTF-8 against field errors, k_heavy against k_copy_rows, across warps and CTAs;
* every decode class through COPY escaping, valid and rejected spellings;
* the Arrow, RowBinary and BigQuery emitters on the heap, window and long-field batches.

first_error is (row, step, code): step 0 = the row's UTF-8 check, 1 + number of fields for an unterminated row,
1 + column otherwise."""
import os
import re

import numpy as np
import pytest

import scenarios as sc
import test_gpu_bigquery as BQ
import test_gpu_rowbinary as RB
from canon import decode_cell
from etl_b200 import abi, pgoutput as pg
from test_gpu_arrow_copy import check_copy_emit, copy_batch, copy_escape, kinds_of, oracle_rows
from test_gpu_copy import BOOL, BYTEA, DATE, FLOAT8, IN_HEAP, INT4, INT8, JSONB, NUMERIC, ORC2ETL, TEXT, TSTZ, UUID, cols_of, synth_rows
from test_gpu_parity import ARRAY_COLS, FUZZ_KINDS

gpu_only = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
with open(os.path.join(ROOT, "etl_b200", "csrc", "rows_kernel.cuh")) as _f:
    WIN = int(re.search(r"#define ETL_ROWS_WIN (\d+)", _f.read()).group(1))
E_UTF8, E_UUID, E_NOT_TERMINATED = 1, 6, 101
K_NUMERIC, K_UUID, K_BYTES = 9, 14, 16
TEXT_ARRAY = 1009


@pytest.fixture(scope="module")
def gpu():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from etl_b200 import decoder
    return decoder


# ------------------------------------------------------------------------------------------------ comparison
def oracle_expect(oracle_mod, oids, rows, values=True):
    """the oracle, row by row: (first error as (row, step, code) or None, {row: values} of every row it accepts)"""
    err, vals = None, {}
    for i, row in enumerate(rows):
        e, ecol, cells, text, heap = oracle_mod.parse_copy_row(oids, row)
        if e:
            if err is None:
                step = 0 if e == E_UTF8 else (1 + len(cells) if e == E_NOT_TERMINATED else 1 + ecol)
                err = (i, step, ORC2ETL.get(e, e))
        elif values:
            vals[i] = [decode_cell(t, v, a, text, heap) for t, v, a in cells]
    return err, vals


def device_values(b, rows):
    heap, stream = b.heap.tobytes(), b.stream.tobytes()
    tags, vals, auxs = b.cell_tag.tolist(), b.cell_val.tolist(), b.cell_aux.tolist()
    out = {}
    for r in rows:
        vs = []
        for i in range(r * b.n_cols, (r + 1) * b.n_cols):
            t, v, a = tags[i], vals[i], auxs[i]
            if t in (2, 15) and v & IN_HEAP:
                vs.append(decode_cell(t, v & ~IN_HEAP, a, heap, heap))
            else:
                vs.append(decode_cell(t, v, a, stream, heap))
        out[r] = vs
    return out


def device_decode(gpu, oids, rows, dec=None):
    own = dec is None
    if own:
        dec = gpu.Decoder(0)
    dec.put_table_schema(7, cols_of(oids))
    try:
        return dec.copy_decode(7, rows)
    finally:
        if own:
            dec.close()


def first_error(b):
    return None if b.first_error[0] is None else tuple(b.first_error[:3])


def check_rows(gpu, oracle_mod, oids, rows, what, labels=None, dec=None, expect_error=None):
    """one batch: first_error and the value of every row the oracle accepts (also those after a failing row).
    `labels[r]` names what row r probes; `expect_error`: False / True / None = the inputs must be valid / must fail / either"""
    want_err, want = oracle_expect(oracle_mod, oids, rows)
    if expect_error is not None:
        assert (want_err is not None) == expect_error, (what, want_err)
    b = device_decode(gpu, oids, rows, dec)
    assert first_error(b) == want_err, (what, first_error(b), want_err, labels[want_err[0]] if labels and want_err else None)
    got = device_values(b, want.keys())
    for r, w in want.items():
        if got[r] != w:
            raise AssertionError(f"{what}: row {r} ({labels[r] if labels else rows[r][:60]!r}): {got[r]} != {w}")
    return want_err


def check_bulk(gpu, oracle_mod, oids, rows, what):
    """a large batch: canonical digest of the valid prefix, first_error from the failing row's own parse"""
    n = len(rows)
    offs = np.zeros(n + 1, dtype=np.uint64)
    offs[1:] = np.cumsum([len(r) for r in rows])
    buf = np.frombuffer(b"".join(rows), dtype=np.uint8)
    digest, err = oracle_mod.copy_rows_digest(oids, buf, offs)
    want_err = None if err is None else oracle_expect(oracle_mod, oids, [rows[err[0]]], values=False)[0]
    want_err = None if want_err is None else (err[0],) + want_err[1:]
    dec = gpu.Decoder(0)
    dec.put_table_schema(7, cols_of(oids))
    b = dec.copy_decode(7, buf, offs)
    dec.close()
    assert first_error(b) == want_err, (what, first_error(b), want_err)
    n_ok = n if err is None else err[0]
    assert oracle_mod.copy_planes_digest(b.cell_tag, b.cell_val, b.cell_aux, n_ok, len(oids), b.stream, b.heap) == digest, what
    return want_err


def check_emitters(gpu, oracle_mod, oids, rows, what):
    """Arrow (plain, ALL | CDC), RowBinary and BigQuery of one COPY batch against their restatements on the oracle's rows"""
    lib = abi.load()
    kinds = kinds_of(oracle_mod, oids)
    dec = gpu.Decoder(0)
    dec.put_table_schema(7, cols_of(oids))
    with copy_batch(gpu, dec, 7, rows) as bh:
        want = oracle_rows(oracle_mod, oids, rows)
        assert check_copy_emit(lib, bh, kinds, want, what) == len(want)
        flags = [True] * (len(oids) + 2)
        rc, h = RB.rb_emit(lib, bh, 0, flags)
        assert rc == 0, (what, rc)
        try:
            RB.check(lib, h, RB.copy_want(oracle_mod, oids, rows, flags), f"{what} (RowBinary)")
        finally:
            lib.etl_dec_rowbinary_free(h)
        rc, h = BQ.bq_emit(lib, bh, 0)
        assert rc == 0, (what, rc)
        try:
            BQ.check(lib, h, BQ.copy_want(oracle_mod, oids, rows), f"{what} (BigQuery)", len(oids), streaming=False)
        finally:
            lib.etl_dec_bigquery_free(h)
    dec.close()


# ------------------------------------------------------------------------------------------------ heap sizing
SHORT_ESC = [b"\\\\", b"\\t", b"\\n", b"\\\\N", b"\\r", b"a\\\\"]


def _heap_text(n, rng):
    return [TEXT], [SHORT_ESC[int(rng.integers(0, len(SHORT_ESC)))] + b"\n" for _ in range(n)]


def _heap_int4_text(n, rng):
    return [INT4, TEXT], [b"%d\t%s\n" % (int(rng.integers(0, 100)), SHORT_ESC[int(rng.integers(0, len(SHORT_ESC)))]) for _ in range(n)]


def _heap_text8(n, rng):
    pool = SHORT_ESC + [b"\\N", b"", b"q"]
    return [TEXT] * 8, [b"\t".join(pool[int(k)] for k in rng.integers(0, len(pool), size=8)) + b"\n" for _ in range(n)]


def _heap_heavy(n, rng):
    """escaped json / numeric / float / bytea: k_heavy parses them from their heap copy"""
    docs = [b'"\\\\n"', b'["\\\\t", 1]', b'{"k": "a\\\\\\\\b"}', b'"\\\\u00e9"']
    nums = [b"\\1", b"1\\.5", b"-\\0", b"\\N\\a\\N", b"12\\3.4\\5"]
    floats = [b"\\1", b"-\\2.5e\\3", b"\\i\\nf", b"N\\aN"]
    out = []
    for _ in range(n):
        f = [docs[int(rng.integers(0, len(docs)))], nums[int(rng.integers(0, len(nums)))], floats[int(rng.integers(0, len(floats)))],
             SHORT_ESC[int(rng.integers(0, len(SHORT_ESC)))], b"\\\\x" + bytes(rng.integers(0, 256, size=int(rng.integers(0, 3)), dtype=np.uint8)).hex().encode()]
        out.append(b"\t".join(f) + b"\n")
    return [JSONB, NUMERIC, FLOAT8, TEXT, BYTEA], out


def _heap_uuid_short(n, rng):
    """empty and 1-byte uuid fields (declined by the light pass: a slot in k_copy_rows and one in k_heavy), one valid
    uuid in 32 rows"""
    import uuid as _uuid
    out = []
    for r in range(n):
        if r % 32 == 5:
            out.append(str(_uuid.UUID(int=int(rng.integers(0, 2**62)) << 64 | int(rng.integers(0, 2**62)))).encode() + b"\n")
        else:
            out.append((b"" if rng.integers(0, 2) else b"%x" % int(rng.integers(0, 16))) + b"\n")
    return [UUID], out


HEAP_CORPORA = {"text": _heap_text, "int4_text": _heap_int4_text, "text8": _heap_text8, "heavy": _heap_heavy, "uuid_short": _heap_uuid_short}
# corpora that need more than the scalar heap etl_dec_copy_decode used to reserve
OLD_BOUND_EXCEEDED = {"text", "int4_text", "text8", "uuid_short"}


def heap_corpus(name, n):
    return HEAP_CORPORA[name](n, np.random.default_rng(1000 + n + len(name)))


def _unescape(raw):
    out, i = bytearray(), 0
    while i < len(raw):
        c = raw[i]
        if c == 0x5C and i + 1 < len(raw):
            i += 1
            c = raw[i]
            if c == ord("N"):
                out += b"\\"
            else:
                c = {ord("b"): 8, ord("f"): 12, ord("n"): 10, ord("r"): 13, ord("t"): 9, ord("v"): 11}.get(c, c)
        elif c == 0x5C:
            i += 1
            continue
        out.append(c)
        i += 1
    return bytes(out)


def _fields(row):
    """raw bytes of every terminated field of a COPY row (TAB / LF ends a field unless escaped)"""
    out, cur, esc = [], bytearray(), False
    for c in row:
        if esc:
            cur.append(c)
            esc = False
        elif c in (9, 10):
            out.append(bytes(cur))
            cur = bytearray()
        else:
            cur.append(c)
            esc = c == 0x5C
    return out


def _cell_heap_bound(kind, n):
    if kind == K_NUMERIC:
        return (8 + 2 * (n // 4 + 2) + 7) & ~7
    if kind == K_BYTES:
        return (((n - 2) // 2 + 7) & ~7) if n >= 2 else 0
    return 16 if kind == K_UUID else 0


def heap_need(kinds, rows):
    """scalar heap bytes k_copy_rows and k_heavy bump-allocate for these rows (restated from the kernels)"""
    need = 0
    for row in rows:
        for k, raw in zip(kinds, _fields(row)):
            if b"\\" in raw:
                if raw == b"\\N":
                    continue
                need += (len(raw) + 7) & ~7                      # the unescaped copy
                text = _unescape(raw)
                if text != b"\\N":
                    need += _cell_heap_bound(k, len(text))
            elif k == K_UUID:
                need += 16 + (16 if len(raw) != 36 else 0)      # slot of the light pass; k_heavy's when it declined
            else:
                need += _cell_heap_bound(k, len(raw))
    return need


def copy_heap_bounds(kinds, rows):
    """(the scalar heap etl_dec_copy_decode reserved before, the one it reserves now) for a batch"""
    ln, nc = sum(len(r) for r in rows), len(rows) * len(kinds)
    any_heap = any(k in (K_NUMERIC, K_UUID, K_BYTES) or k & 0x20 for k in kinds)
    old = ln + 64 + ((ln // 2 + 24 * nc + 256) if any_heap else 0)
    new = ln + 8 * nc + 64 + ((ln // 2 + 32 * nc + 256) if any_heap else 0)
    return (old + 15) & ~15, (new + 15) & ~15


@pytest.mark.parametrize("name", sorted(HEAP_CORPORA))
def test_heap_corpora_stress_the_bound(oracle_mod, name):
    """CPU: the heap corpora need more heap than their input length + 64, the ones meant to overflow the former
    reservation do, and the current reservation holds them"""
    for n in (1, 13, 1000, 100000):
        oids, rows = heap_corpus(name, n)
        kinds = kinds_of(oracle_mod, oids)
        need, ln = heap_need(kinds, rows), sum(len(r) for r in rows)
        old, new = copy_heap_bounds(kinds, rows)
        assert need <= new, (name, n, need, new)
        if n >= 1000:
            assert need > ln + 64, (name, n, need, ln)
            assert (need > old) == (name in OLD_BOUND_EXCEEDED), (name, n, need, old)


@gpu_only
@pytest.mark.parametrize("n", [1, 13, 1000, 100000])
@pytest.mark.parametrize("name", sorted(HEAP_CORPORA))
def test_heap_corpora(gpu, oracle_mod, name, n):
    oids, rows = heap_corpus(name, n)
    if n <= 1000:
        check_rows(gpu, oracle_mod, oids, rows, f"{name} x {n}")
    else:
        check_bulk(gpu, oracle_mod, oids, rows, f"{name} x {n}")


@gpu_only
def test_valid_uuids_then_short_ones(gpu, oracle_mod):
    """5 000 valid uuid rows, then 5 000 with empty or 1-byte fields: the first short one is the error, the valid
    prefix is exact"""
    import uuid as _uuid
    rng = np.random.default_rng(77)
    rows = [str(_uuid.UUID(bytes=bytes(rng.integers(0, 256, size=16, dtype=np.uint8)))).encode() + b"\n" for _ in range(5000)]
    rows += [(b"" if r % 2 else b"f") + b"\n" for r in range(5000)]
    assert check_bulk(gpu, oracle_mod, [UUID], rows, "uuid 5000 + 5000") == (5000, 1, E_UUID)


UUID_COLS = [sc.col("id", sc.INT8, 1)] + [sc.col(f"u{i}", UUID, None, True) for i in range(16)]
UUID_RECORDS = 20000


def uuid_stream(bad):
    rel = pg.relation(96, "public", "uuids", "d", sc.rel_cols(UUID_COLS, {"id"}))
    w = pg.StreamWriter()
    tx = sc.Tx(w)
    tx.begin()
    w.emit(rel)
    for r in range(UUID_RECORDS):
        vals = [("" if (r + i) % 3 else "z") for i in range(16)] if bad else ["a0eebc99-9c0b-4ef8-bb6d-6bb9bd3%05d" % ((r * 16 + i) % 100000) for i in range(16)]
        w.emit(pg.insert(96, [str(r)] + vals))
    tx.commit()
    return w.bytes()


def test_replication_uuid_stream_stresses_the_bound():
    """CPU: 32 bytes per declined uuid cell is more than the replication path's former scalar heap (len/2 + 24 per cell)
    and within the current one"""
    ln, n_cells = len(uuid_stream(True)), UUID_RECORDS * len(UUID_COLS)
    need = 32 * 16 * UUID_RECORDS
    assert ln // 2 + 24 * n_cells + 256 < need <= ln // 2 + 32 * n_cells + 256


@gpu_only
def test_replication_declined_uuids(gpu, oracle_mod):
    """the replication path: records of 16 uuid columns holding short invalid values (a heap slot in k_rows and one in
    k_heavy for each), first_error compared; a clean stream of the same shape compared plane by plane"""
    from canon import assert_planes_equal
    cols = UUID_COLS
    for bad in (True, False):
        stream = uuid_stream(bad)
        dec, orc = gpu.Decoder(0), oracle_mod.Oracle()
        dec.put_table_schema(96, cols)
        orc.put_table_schema(96, cols)
        got, want = dec.decode(stream), orc.decode(stream)
        dec.close()
        assert (want.first_error[0] is not None) == bad
        assert got.first_error == want.first_error, (got.first_error, want.first_error)
        if not bad:
            assert_planes_equal(got, want, stream)


# ------------------------------------------------------------------------------------------------ window edges
EDGE_TABLES = {"text": [TEXT, TEXT, TEXT], "mixed": [INT8, TEXT, NUMERIC, TEXT]}
UTF8_4 = "\U0001F914".encode()


def _probe(table, feature, o):
    """a valid row of `table` whose `feature` starts at row offset o"""
    if table == "text":
        head, tail = b"", b"\tb\tc\n"
    else:
        head, tail = b"12\t", b"\t1.5\tz\n"
    fill = o - len(head)
    if feature == "tab":                                  # ends the long field
        return head + b"a" * fill + tail
    if feature == "lf":                                   # ends the row
        pre = b"a\tb\t" if table == "text" else b"12\tx\t1.5\t"
        return pre + b"c" * (o - len(pre)) + b"\n"
    if feature in ("backslash", "esc_tab", "esc_lf", "esc_t", "utf8"):
        f = {"backslash": b"\\\\", "esc_tab": b"\\\t", "esc_lf": b"\\\n", "esc_t": b"\\t", "utf8": UTF8_4}[feature]
        return head + b"a" * fill + f + b"a" + tail
    if feature == "null":                                 # `\N` as the field after the long one
        return head + b"a" * (fill - 1) + b"\t\\N" + (b"\tc\n" if table == "text" else b"\tz\n")
    if feature == "digits":                               # a light / heavy value spanning the offset
        if table == "text":
            return b"a" * (o - 4) + b"\tbbbbbbbb\tc\n"
        return b"0" * o + b"7\tx\t-000000123.4500\tz\n" if o % 2 else b"1\t" + b"a" * (o - 6) + b"\t1234567.891\tz\n"
    raise ValueError(feature)


EDGE_FEATURES = ["tab", "lf", "backslash", "esc_tab", "esc_lf", "esc_t", "null", "utf8", "digits"]


def _filler(table, length):
    pre = b"x\ty\t" if table == "text" else b"1\tx\t2\t"
    return pre + b"z" * (length - len(pre) - 1) + b"\n"


def edge_batch(table):
    """probe rows for every (row start mod 16, feature, window end 1 / 2, offset -24..24), each after a filler row that
    puts its start at that residue; window end k lies at k * WIN - (row start mod 16) from the row start"""
    rows, labels, at = [], [], 0
    min_fill = 8
    for a in range(16):
        for feature in EDGE_FEATURES:
            for k in (1, 2):
                for d in range(-24, 25):
                    ln = min_fill + (a - at - min_fill) % 16
                    rows.append(_filler(table, ln))
                    labels.append("filler")
                    at += ln
                    assert at % 16 == a
                    r = _probe(table, feature, k * WIN - a + d)
                    rows.append(r)
                    labels.append(f"{feature} at window end {k} {d:+d}, row start = {a} mod 16")
                    at += len(r)
    return rows, labels


@gpu_only
@pytest.mark.parametrize("table", sorted(EDGE_TABLES))
def test_window_edges(gpu, oracle_mod, table):
    rows, labels = edge_batch(table)
    check_rows(gpu, oracle_mod, EDGE_TABLES[table], rows, f"window edges ({table})", labels, expect_error=False)
    # a share of the probes alone behind one filler row (same residue), where no other lane moves the window
    dec = gpu.Decoder(0)
    try:
        for i in range(1, len(rows), 50):
            a = int(re.search(r"= (\d+) mod 16", labels[i]).group(1))
            check_rows(gpu, oracle_mod, EDGE_TABLES[table], [_filler(table, 8 + (a - 8) % 16), rows[i]], f"{labels[i]} alone",
                       ["filler", labels[i]], dec=dec, expect_error=False)
    finally:
        dec.close()


# ------------------------------------------------------------------------------------------------ long fields
LONG_OIDS = [INT4, INT8, TEXT, NUMERIC, FLOAT8, JSONB, BYTEA, TEXT_ARRAY]
SHORT_VALUES = [b"7", b"-8", b"short", b"1.5", b"2.5", b'{"a": 1}', b"\\\\x00ff", b"{a,b}"]
HALF_ABOVE_ONE = "1.00000000000000011102230246251565404236316680908203125"   # exactly halfway between 1 and its successor


def long_values(rng):
    """(column, bytes) values longer than a staging window, per decode class, and heavy values around the 128 bytes
    k_heavy stages"""
    utf = "caf\u00e9 \u6d4b\u8bd5 \U0001F914 ".encode()
    text = (b"".join(rng.choice([b"abc", b"\\t", b"\\\\", b"\\n", utf, b"x" * 40], size=600)))[:5000]
    out = [(0, b"0" * 500 + b"42"), (0, b"-" + b"0" * 500 + b"2147483648"), (1, b"0" * 500 + b"9223372036854775807"),
           (1, b"-" + b"0" * 500 + b"9223372036854775808"), (2, text), (2, b"y" * 5000),
           (3, b"9" * 600 + b"." + b"1" * 400), (3, b"-0." + b"0" * 998 + b"1"),
           (4, (HALF_ABOVE_ONE + "0" * 800).encode()), (4, (HALF_ABOVE_ONE + "0" * 800 + "1").encode()),
           (4, ("0." + "0" * 300 + "4940656458412465441765687928682213723651" + "7" * 500 + "e+1").encode()),
           (5, b'{"k": [' + b",".join(b'"v%d\\\\t"' % i if i % 7 == 0 else b"%d" % i for i in range(16000)) + b"]}"),
           (6, b"\\\\x" + bytes(rng.integers(0, 256, size=65536, dtype=np.uint8)).hex().encode()),
           (7, b"{" + b",".join(b'"e\\\\\\\\%d"' % i if i % 5 == 0 else b"w%d" % i for i in range(2500)) + b"}")]
    for ln in range(120, 137, 2):                          # heap copies that k_heavy stages or reads directly
        out.append((3, b"\\1" + b"2" * (ln - 1)))
        out.append((5, b'"' + b"j" * (ln - 5) + b'\\\\n"'))
        out.append((4, b"\\1." + b"0" * (ln - 2)))
    return out


def long_batch():
    rng = np.random.default_rng(9)
    rows = []
    for c, v in long_values(rng):
        for pos in range(3):                               # the long row in lane 0, 1 and 2 of its warp among short rows
            f = list(SHORT_VALUES)
            f[c] = v
            for _ in range(pos):
                rows.append(b"\t".join(SHORT_VALUES) + b"\n")
            rows.append(b"\t".join(f) + b"\n")
    return LONG_OIDS, rows


@gpu_only
def test_long_fields(gpu, oracle_mod):
    oids, rows = long_batch()
    check_rows(gpu, oracle_mod, oids, rows, "long fields", expect_error=False)
    for r in rows[:: 7]:                                   # alone in a batch too
        check_rows(gpu, oracle_mod, oids, [r], "long field alone")


# ------------------------------------------------------------------------------------------------ warp divergence
ALTERNATING = [INT4, NUMERIC, TEXT, JSONB, INT8, FLOAT8, BOOL, BYTEA, UUID, TSTZ, DATE, 700]


def alternating_rows(n, seed, long_every=0, long_len=0):
    import uuid as _uuid
    rng = np.random.default_rng(seed)
    rows = []
    for r in range(n):
        t = "".join(rng.choice(list("abc xyz\u00e9"), size=int(rng.integers(0, 20))))
        if long_every and r % long_every == 0:
            t = ("L" * long_len)[:long_len]
        f = [str(int(rng.integers(-10**9, 10**9))), "%d.%d" % (int(rng.integers(0, 10**6)), int(rng.integers(0, 100))),
             copy_escape(t).decode(), copy_escape('{"r": %d, "t": "a\\tb"}' % r).decode(), str(int(rng.integers(-2**62, 2**62))),
             repr(float(rng.standard_normal())), "t" if r % 2 else "f", "\\\\x%02x" % (r % 256),
             str(_uuid.UUID(int=r * 7919 + 1)), "2024-05-%02d 01:02:03.5+00" % (1 + r % 28), "2023-%02d-01" % (1 + r % 12), "%.3f" % (r / 7)]
        for c in range(1, len(f)):
            if rng.integers(0, 15) == 0:
                f[c] = "\\N"
        rows.append(("\t".join(f) + "\n").encode())
    return rows


@gpu_only
@pytest.mark.parametrize("n", [31, 32, 33, 127, 128, 129])
def test_batch_sizes_around_warps_and_ctas(gpu, oracle_mod, n):
    oids, rows = synth_rows(n, 55 + n)
    check_rows(gpu, oracle_mod, oids, rows, f"synthetic x {n}", expect_error=False)
    check_rows(gpu, oracle_mod, ALTERNATING, alternating_rows(n, n), f"alternating classes x {n}", expect_error=False)


@gpu_only
def test_long_rows_among_short_ones(gpu, oracle_mod):
    rows = alternating_rows(96, 3)
    for at in (0, 17, 31, 32, 63, 95):                     # one 10 KiB row at a time, at warp edges and inside a warp
        r = list(rows)
        r[at] = alternating_rows(1, 4, long_every=1, long_len=10240)[0]
        check_rows(gpu, oracle_mod, ALTERNATING, r, f"10 KiB row at {at}", expect_error=False)
    check_rows(gpu, oracle_mod, ALTERNATING, alternating_rows(128, 5, long_every=2, long_len=700), "alternating long / short", expect_error=False)
    check_rows(gpu, oracle_mod, ALTERNATING, alternating_rows(128, 6, long_every=3, long_len=3000), "long every third row", expect_error=False)


@gpu_only
def test_field_counts_differ_within_a_warp(gpu, oracle_mod):
    oids = [INT4, TEXT, INT8]
    rows = [b"1\ta\t2\n"] * 128
    for r, row in ((7, b"1\ta\t2\t3\n"), (8, b"1\ta\n"), (9, b"1\ta\t2\t\n"), (40, b"1\n"), (41, b"1\ta\t2\tx\ty\n"), (100, b"\t\t\t\t\n")):
        rows[r] = row
    for k in range(128):                                   # a long field now and then, so that some lanes restage
        if k % 5 == 2 and rows[k] == b"1\ta\t2\n":
            rows[k] = b"1\t" + b"w" * 900 + b"\t2\n"
    assert check_rows(gpu, oracle_mod, oids, rows, "n_cols - 1 / n_cols / n_cols + 1 fields") == (7, 4, 26)
    rows2 = list(rows)
    rows2[7] = rows2[9] = b"1\ta\t2\n"
    assert check_rows(gpu, oracle_mod, oids, rows2, "too few first") == (8, 3, 26)


# ------------------------------------------------------------------------------------------------ column counts
CYCLE = [INT4, TEXT, NUMERIC, BOOL, JSONB, UUID, FLOAT8, INT8, DATE]
CYCLE_VALUES = {INT4: ["5", "-17", "\\N"], TEXT: ["t", "a\\tb", ""], NUMERIC: ["1.25", "NaN", "\\N"], BOOL: ["t", "f"], JSONB: ["[1]", '{"a": "\\\\n"}'],
                UUID: ["a0eebc99-9c0b-4ef8-bb6d-6bb9bd380a11", "A0EEBC999C0B4EF8BB6D6BB9BD380A11"], FLOAT8: ["1e5", "-0.5"],
                INT8: ["9223372036854775807", "0"], DATE: ["2024-02-29", "1999-12-31"]}
BAD = {INT4: "x", TEXT: None, NUMERIC: "1.2.3", BOOL: "yes", JSONB: "{", UUID: "zz", FLOAT8: "1e", INT8: "9223372036854775808", DATE: "2023-02-29"}


def wide_rows(n_cols, n_rows, seed):
    oids = [CYCLE[c % len(CYCLE)] for c in range(n_cols)]
    rng = np.random.default_rng(seed)
    rows = []
    for _ in range(n_rows):
        rows.append(("\t".join(CYCLE_VALUES[o][int(rng.integers(0, len(CYCLE_VALUES[o])))] for o in oids) + "\n").encode())
    return oids, rows


@gpu_only
@pytest.mark.parametrize("n_cols", [1, 255, 256, 257, 300, 1600])
def test_column_counts(gpu, oracle_mod, n_cols):
    oids, rows = wide_rows(n_cols, 70, n_cols)
    check_rows(gpu, oracle_mod, oids, rows, f"{n_cols} columns", expect_error=False)
    fields = [r[:-1].split(b"\t") for r in rows]
    last = max(c for c in range(n_cols) if BAD[oids[c]] is not None)
    cases = []
    f = list(fields[33])
    f[last] = BAD[oids[last]].encode()
    cases.append((33, b"\t".join(f) + b"\n", 1 + last))                  # a field error in the last checkable column
    cases.append((40, b"\t".join(fields[40] + [b"1"]) + b"\n", 1 + n_cols))   # one field too many
    if n_cols > 1:
        cases.append((45, b"\t".join(fields[45][:-1]) + b"\n", n_cols))       # one too few
    for at, row, step in cases:
        r = list(rows)
        r[at] = row
        err = check_rows(gpu, oracle_mod, oids, r, f"{n_cols} columns, error case at step {step}")
        assert err[:2] == (at, step), err


@gpu_only
def test_zero_columns(gpu, oracle_mod):
    dec = gpu.Decoder(0)
    dec.put_table_schema(8, [])
    b = dec.copy_decode(8, [])
    assert first_error(b) is None and b.n_rows == 0
    b = dec.copy_decode(8, [b"\n", b"\n"])
    dec.close()
    assert first_error(b) == oracle_expect(oracle_mod, [], [b"\n", b"\n"])[0] == (0, 1, 26)


ODD_ROWS = [   # (type oids, rows, whether the oracle must accept every row)
    ([INT4, INT4], [b"1\n2\n"], True),                          # an LF ends a field: two fields, one row
    ([INT4], [b"42\ntrailing"], True),                          # bytes after the last LF are dropped
    ([TEXT, TEXT], [b"a\tb\n\\"], True),
    ([TEXT, TEXT], [b"a\tb\nc\td\te"], False),           # fields after the LF still count
    ([TEXT], [b""], False),                                     # an empty row
    ([TEXT], [b"abc\\\n"], False),                              # its only LF is escaped
    ([TEXT], [b"abc\\"], False),                                # a trailing lone backslash
    ([TEXT, INT4], [b"x\t5\\"], False),
    ([INT4], [b"1\r\n"], False),                                # CR before the LF on an int column
    ([TEXT], [b"1\r\n"], True),
    ([TEXT, INT4], [b"a\x00b\t5\n", b"\x00" * 40 + b"\t0\n", b"\x00\\\x00\t1\n"], True),   # NUL bytes inside text
    ([TEXT], [b"\\\\N\n", b"\\N\n", b"\\\\\\N\n", b"N\\\n\n"], True),
]


@gpu_only
@pytest.mark.parametrize("idx", range(len(ODD_ROWS)))
def test_odd_rows(gpu, oracle_mod, idx):
    oids, rows, ok = ODD_ROWS[idx]
    check_rows(gpu, oracle_mod, oids, rows, f"odd rows {idx}", expect_error=not ok)
    pad = [b"\t".join(b"1" for _ in oids) + b"\n"] * 45                     # the same rows inside a batch, in a later warp
    check_rows(gpu, oracle_mod, oids, pad + rows + pad, f"odd rows {idx} in a batch", expect_error=not ok)


# ------------------------------------------------------------------------------------------------ error order
ROW_ERRORS = [   # (type oids, row, expected (step, code))
    ([INT4, TEXT], b"x\tabc\n\xff", (0, 1)),                    # invalid UTF-8 after the LF beats a field error
    ([TEXT, INT4], b"a\\\xff\tx\n", (0, 1)),                    # ... inside an escape
    ([INT4, TEXT], b"x\tab\xc3", (0, 1)),                       # ... in unterminated trailing bytes
    ([INT4, TEXT], b"x\tab\n\xc3\xa9z", (1, 2)),                # valid UTF-8 there: the field error
    ([NUMERIC, INT4], b"1.2.3\tx\n", (1, 5)),                   # k_heavy's error in an earlier column
    ([JSONB, BOOL], b"{bad\tq\n", (1, 7)),
    ([FLOAT8, UUID], b"1e\tzz\n", (1, 3)),
    ([INT4, NUMERIC], b"x\t1.2.3\n", (1, 2)),                   # light error first
    ([BOOL, JSONB, INT4], b"t\t{\tx\n", (2, 7)),
    ([INT4, INT4], b"x\t1\t2\n", (1, 2)),                       # a parse error before one field too many
    ([INT4, INT4, INT4], b"1\tx\n", (2, 2)),                    # ... before too few fields
    ([NUMERIC, INT4], b"1.2.3\t1\t2\n", (1, 5)),
    ([INT4], b"1\t2\tx\n", (2, 26)),                            # the first extra field ends the row's columns
    ([JSONB, TEXT], b"[\tx", (1, 7)),                           # a field error before "not terminated"
    ([JSONB, TEXT], b"[1]\tx", (2, 25)),
]


@gpu_only
@pytest.mark.parametrize("idx", range(len(ROW_ERRORS)))
def test_error_order_within_a_row(gpu, oracle_mod, idx):
    oids, row, (step, code) = ROW_ERRORS[idx]
    assert check_rows(gpu, oracle_mod, oids, [row], f"row error {idx}") == (0, step, code)
    good = b"\t".join({INT4: b"1", TEXT: b"t", NUMERIC: b"2.5", JSONB: b"[]", BOOL: b"t", FLOAT8: b"1", UUID: b"a0eebc99-9c0b-4ef8-bb6d-6bb9bd380a11"}[o]
                      for o in oids) + b"\n"
    assert check_rows(gpu, oracle_mod, oids, [good] * 70 + [row] + [good] * 60, f"row error {idx} in a batch") == (70, step, code)


ACROSS = [NUMERIC, INT4, JSONB, TEXT]


def _across(errors, n=300):
    """rows of ACROSS (4 CTAs of k_copy_rows), valid except {row: [(column, bad value)] or the whole row}"""
    rows = []
    for r in range(n):
        e = errors.get(r, [])
        if isinstance(e, bytes):
            rows.append(e)
            continue
        f = [b"%d.25" % r, b"%d" % r, b'{"r": %d}' % r, b"t%d" % r]
        for c, v in e:
            f[c] = v
        rows.append(b"\t".join(f) + b"\n")
    return rows


ACROSS_CASES = [   # (errors, expected (row, step, code))
    ({40: [(1, b"x")], 33: [(2, b"{")], 34: [(3, b"\xff")], 200: [(1, b"y")]}, (33, 3, 7)),   # one warp: k_heavy's error, earliest row
    ({33: [(0, b"1.2.3"), (1, b"x")]}, (33, 1, 5)),                                         # one row: k_heavy's error, earlier column
    ({33: [(1, b"x"), (2, b"{")], 32: [(3, b"\xc3")]}, (32, 0, 1)),
    ({149: [(1, b"x")], 150: [(0, b"1..")]}, (149, 2, 2)),                                 # the second CTA
    ({129: [(0, b"nan1")], 260: [(1, b"z")]}, (129, 1, 5)),                               # k_heavy's error in the earlier CTA
    ({129: [(1, b"z")], 260: [(0, b"nan1")]}, (129, 2, 2)),
    ({**{r: [(2, b"[")] for r in range(160, 300, 3)}, 161: [(1, b"q")]}, (160, 3, 7)),    # many rows of several warps
    ({**{r: [(0, b"-")] for r in range(96, 128)}, 95: b"95.25\t95\t{}\tunterminated"}, (95, 4, 25)),   # a row without its LF
]


@gpu_only
@pytest.mark.parametrize("idx", range(len(ACROSS_CASES)))
def test_error_order_across_rows(gpu, oracle_mod, idx):
    errors, want = ACROSS_CASES[idx]
    assert check_rows(gpu, oracle_mod, ACROSS, _across(errors), f"errors across rows {idx}") == want


# ------------------------------------------------------------------------------------------------ every decode class
def fuzz_cases(oid, seeds, alphabet):
    rng = np.random.default_rng(oid + 7)
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
    return list(dict.fromkeys(cases))


def check_class(gpu, oracle_mod, oid, values):
    """valid spellings (by the oracle's verdict on the COPY row) in one batch, every value compared; each rejected one
    alone (at most 60)"""
    oids = [INT8, oid]
    rows = [b"%d\t%s\n" % (i, copy_escape(v)) for i, v in enumerate(values)]
    verdict = [oracle_mod.parse_copy_row(oids, r)[0] == 0 for r in rows]
    valid = [r for r, ok in zip(rows, verdict) if ok]
    assert valid, oid
    check_rows(gpu, oracle_mod, oids, valid, f"oid {oid} valid", expect_error=False)
    dec = gpu.Decoder(0)
    try:
        for r in [r for r, ok in zip(rows, verdict) if not ok][:60]:
            check_rows(gpu, oracle_mod, oids, [r], f"oid {oid} rejected {r!r}", dec=dec, expect_error=True)
    finally:
        dec.close()


@gpu_only
@pytest.mark.parametrize("oid", [k[0] for k in FUZZ_KINDS])
def test_every_scalar_class(gpu, oracle_mod, oid):
    _, seeds, alphabet = next(k for k in FUZZ_KINDS if k[0] == oid)
    check_class(gpu, oracle_mod, oid, fuzz_cases(oid, seeds, alphabet))


@gpu_only
@pytest.mark.parametrize("oid", [k[0] for k in ARRAY_COLS])
def test_every_array_class(gpu, oracle_mod, oid):
    _, good, bad = next(k for k in ARRAY_COLS if k[0] == oid)
    check_class(gpu, oracle_mod, oid, list(good) + list(bad))


# ------------------------------------------------------------------------------------------------ the emitters
@gpu_only
@pytest.mark.parametrize("name", sorted(HEAP_CORPORA))
def test_emitters_on_heap_corpora(gpu, oracle_mod, name):
    oids, rows = heap_corpus(name, 1000)
    check_emitters(gpu, oracle_mod, oids, rows, f"heap corpus {name}")


@gpu_only
@pytest.mark.parametrize("table", sorted(EDGE_TABLES))
def test_emitters_on_window_edges(gpu, oracle_mod, table):
    rows, _ = edge_batch(table)
    check_emitters(gpu, oracle_mod, EDGE_TABLES[table], rows, f"window edges ({table})")


@gpu_only
def test_emitters_on_long_fields(gpu, oracle_mod):
    oids, rows = long_batch()
    check_emitters(gpu, oracle_mod, oids, rows, "long fields")
