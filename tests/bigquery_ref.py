"""Python restatement of the BigQuery destination's Storage Write rows (crates/etl-destinations/src/bigquery):
write_events (core.rs:792-970) choosing the rows and pushing _CHANGE_TYPE / _CHANGE_SEQUENCE_NUMBER,
bigquery_update_rows / bigquery_primary_key_changed (:1255-1403) splitting a primary-key change into DELETE + UPSERT,
bigquery_delete_row (:1406-1524) building sparse key rows, write_table_rows (:530-546) for COPY rows,
try_from_tagged_cells / validate_cell_for_bigquery (encoding.rs:49-83, validation.rs) and the prost serialisation
cell_encode_prost / array_cell_encode_prost (encoding.rs:151-342).

Applied to a decoded batch's planes (canon.decode_cell values), `expected_bigquery` gives what etl_dec_bigquery_emit
must produce: rows, their bytes, the first value issue and the first invalid record.  The reference stops at an issue;
the emitter carries on, so a row with an issue follows the emitter's convention here (a NULL array element writes
nothing), which keeps every later row's offsets comparable.
"""
from __future__ import annotations

import datetime
import struct

from arrow_ref import json_display, numeric_display
from canon import CELL_ARRAY, CELL_NULL, RF_EVENT, RF_NEW_PARTIAL, RF_OLD_FULL, RF_OLD_KEY, decode_cell

NONE64, NONE32 = 2**64 - 1, 2**32 - 1
ISSUE_ARRAY_NULL, ISSUE_NUMERIC_SCALE, ISSUE_JSON_INTEGER = 1, 2, 3
WT_VARINT, WT_I64, WT_LEN, WT_I32 = 0, 1, 2, 5
PACKED = {1, 3, 4, 5, 6, 7, 8}                  # Bool, I16, I32, U32, I64, F32, F64 (cell tags = element kinds)
MAX_SCALE = 38


# ------------------------------------------------------------------------------------------------ wire
def varint(n: int) -> bytes:
    out = bytearray()
    while True:
        b = n & 0x7F
        n >>= 7
        if n == 0:
            out.append(b)
            return bytes(out)
        out.append(b | 0x80)


def key(field: int, wt: int) -> bytes:
    return varint(field << 3 | wt)


def len_field(field: int, payload: bytes) -> bytes:
    return key(field, WT_LEN) + varint(len(payload)) + payload


# ------------------------------------------------------------------------------------------------ text forms
def year_text(y: int) -> str:
    """chrono's %Y: 0..=9999 as 4 digits, else sign and at least 4 digits"""
    return "%04d" % y if 0 <= y <= 9999 else ("-" if y < 0 else "+") + "%04d" % abs(y)


def civil(days: int):
    """proleptic Gregorian date of a day count from 1970-01-01, for any year (datetime stops at 1..9999)"""
    z = days + 719468
    era = z // 146097
    doe = z - era * 146097
    yoe = (doe - doe // 1460 + doe // 36524 - doe // 146096) // 365
    doy = doe - (365 * yoe + yoe // 4 - yoe // 100)
    mp = (5 * doy + 2) // 153
    d = doy - (153 * mp + 2) // 5 + 1
    m = mp + 3 if mp < 10 else mp - 9
    return yoe + era * 400 + (m <= 2), m, d


def date_text(days: int) -> bytes:
    y, m, d = civil(days)
    if 1 <= y <= 9999:
        assert datetime.date(1970, 1, 1) + datetime.timedelta(days=days) == datetime.date(y, m, d)
    return ("%s-%02d-%02d" % (year_text(y), m, d)).encode()


def time_text(secs: int, nanos: int) -> bytes:
    """%H:%M:%S%.f; nanos >= 10^9 is chrono's leap second (:60)"""
    sec = secs % 60
    if nanos >= 10**9:
        sec += 1
        nanos -= 10**9
    out = "%02d:%02d:%02d" % (secs // 3600, secs // 60 % 60, sec)
    if nanos == 0:
        pass
    elif nanos % 10**6 == 0:
        out += ".%03d" % (nanos // 10**6)
    elif nanos % 1000 == 0:
        out += ".%06d" % (nanos // 1000)
    else:
        out += ".%09d" % nanos
    return out.encode()


def timestamp_text(secs: int, nanos: int, tz: bool) -> bytes:
    days, sod = divmod(secs, 86400)
    return date_text(days) + b" " + time_text(sod, nanos) + (b"+00:00" if tz else b"")


def uuid_text(hex32: str) -> bytes:
    h = hex32.lower()
    return ("%s-%s-%s-%s-%s" % (h[:8], h[8:12], h[12:16], h[16:20], h[20:])).encode()


def sequence_key(commit_lsn: int, tx_ordinal: int, ordinal: int) -> bytes:
    """bigquery_sequence_key (core.rs:1235)"""
    return ("%016x/%016x/%016x" % (commit_lsn, tx_ordinal, ordinal)).encode()


# ------------------------------------------------------------------------------------------------ checks
def numeric_scale_bad(num) -> bool:
    """validate_numeric_for_bigquery: Display with more than 38 fractional digits"""
    s = numeric_display(num)
    return len(num) != 2 and len(s.split(".", 1)[1]) > MAX_SCALE if "." in s else False


def json_int_literal_bad(tok: str) -> bool:
    if any(c in tok for c in ".eE"):
        return False
    v = int(tok)
    return not (-2**63 <= v < 2**63) if tok.startswith("-") else not (0 <= v < 2**64)


def json_int_bad(text: bytes) -> bool:
    """validate_json_for_bigquery over every number of the document"""
    import json
    found = []
    json.loads(text.decode("utf-8"), parse_int=lambda t: found.append(t) or 0, parse_float=lambda t: 0.0)
    return any(json_int_literal_bad(t) for t in found)


# ------------------------------------------------------------------------------------------------ values
def text_of(tag: int, v) -> bytes:
    """the UTF-8 text (or Bytes payload) of a non-NULL value of a length-delimited kind"""
    if tag == 2:
        return v.encode("utf-8")
    if tag == 9:
        return numeric_display(v).encode()
    if tag == 10:
        return date_text(v[1])
    if tag == 11:
        return time_text(v[1], v[2])
    if tag == 12:
        return timestamp_text(v[1], v[2], False)
    if tag == 13:
        return timestamp_text(v[1], v[2], True)
    if tag == 14:
        return uuid_text(v[1])
    if tag == 15:
        return json_display(v[1])
    if tag == 16:
        return v[1]
    raise ValueError(f"cell tag {tag} is not length-delimited")


def packed_value(tag: int, v) -> bytes:
    if tag == 1:
        return bytes([int(v)])
    if tag in (3, 4, 6):
        return varint(v & NONE64)
    if tag == 5:
        return varint(v[1])
    if tag == 7:
        return struct.pack("<I", v[1])
    if tag == 8:
        return struct.pack("<Q", v[1])
    raise ValueError(tag)


def scalar_wt(tag: int) -> int:
    return WT_I32 if tag == 7 else (WT_I64 if tag == 8 else WT_VARINT)


def cell_issue(tag: int, v):
    """(kind, element) of a cell's first issue, None if it has none: a NULL element first, then the checks"""
    if tag == 9:
        return (ISSUE_NUMERIC_SCALE, NONE32) if numeric_scale_bad(v) else None
    if tag == 15:
        return (ISSUE_JSON_INTEGER, NONE32) if json_int_bad(v[1]) else None
    if tag == CELL_ARRAY:
        _, ek, elems = v
        for k, e in enumerate(elems):
            if e is None:
                return (ISSUE_ARRAY_NULL, k)
        for k, e in enumerate(elems):
            if ek == 9 and numeric_scale_bad(e):
                return (ISSUE_NUMERIC_SCALE, k)
            if ek == 15 and json_int_bad(e[1]):
                return (ISSUE_JSON_INTEGER, k)
    return None


def field_bytes(field: int, tag: int, v) -> bytes:
    """cell_encode_prost of one cell under `field` (NULL writes nothing; NULL elements are left out)"""
    if tag == CELL_NULL:
        return b""
    if tag == CELL_ARRAY:
        _, ek, elems = v
        if not elems:
            return b""
        vals = [e for e in elems if e is not None]
        if ek in PACKED:
            return len_field(field, b"".join(packed_value(ek, e) for e in vals))
        return b"".join(len_field(field, text_of(ek, e)) for e in vals)
    if tag in PACKED:
        return key(field, scalar_wt(tag)) + packed_value(tag, v)
    return len_field(field, text_of(tag, v))


def row_bytes(tagged, issues: dict, row: int) -> bytes:
    """one message: tagged = [(field, column or None, (tag, value))] in field order; records the first value issue"""
    out = []
    for field, col, (tag, v) in tagged:
        if col is not None and issues.get("value") is None:
            x = cell_issue(tag, v)
            if x is not None:
                issues["value"] = (row, col, x[1], x[0])
        out.append(field_bytes(field, tag, v))
    return b"".join(out)


# ------------------------------------------------------------------------------------------------ key comparison
def cells_equal(a, b) -> bool:
    """Cell's derived PartialEq on decode_cell values: (tag, value)"""
    (ta, va), (tb, vb) = a, b
    if ta != tb:
        return False
    if ta == CELL_ARRAY:
        if va[1] != vb[1] or len(va[2]) != len(vb[2]):
            return False
        return all((x is None and y is None) or (x is not None and y is not None and cells_equal((va[1], x), (vb[1], y)))
                   for x, y in zip(va[2], vb[2]))
    if ta == 7:
        return struct.unpack("<f", struct.pack("<I", va[1]))[0] == struct.unpack("<f", struct.pack("<I", vb[1]))[0]
    if ta == 8:
        return struct.unpack("<d", struct.pack("<Q", va[1]))[0] == struct.unpack("<d", struct.pack("<Q", vb[1]))[0]
    if ta == 15:
        return json_display(va[1]) == json_display(vb[1])
    return va == vb


# ------------------------------------------------------------------------------------------------ rows of a batch
def pk_columns(schema, table_cols):
    return [table_cols[int(i)].get("pk") is not None for i in schema.col_index]


def expected_bigquery(p, stream: bytes, schema_index: int, table_cols):
    """etl_dec_bigquery_emit of a streaming batch's schema version: dict(records, rows, value, invalid)"""
    sc = p.schemas[schema_index]
    heap = p.heap.tobytes()
    nc = sc.n_cols
    pk = pk_columns(sc, table_cols)
    pk_idx = [c for c in range(nc) if pk[c]]
    identity_is_pk = all(bool(int(f) & 2) == pk[c] for c, f in enumerate(sc.col_flags))
    n = p.n_records if p.first_error[0] is None else p.first_error[0]

    def cell(i):
        tag = int(p.cell_tag[i])
        return tag, decode_cell(tag, int(p.cell_val[i]), int(p.cell_aux[i]), stream, heap)

    records, rows, issues, invalid = [], [], {}, NONE64

    def emit(r, tagged, op, ordinal):
        tagged = list(tagged) + [(nc + 1, None, (2, op)),
                                 (nc + 2, None, (2, sequence_key(int(p.rec_commit_lsn[r]), int(p.rec_tx_ordinal[r]), ordinal).decode()))]
        rows.append(row_bytes(tagged, issues, len(rows)))
        records.append(r)

    for r in range(n):
        if int(p.rec_schema[r]) != schema_index or not int(p.rec_flags[r]) & RF_EVENT:
            continue
        k, f = int(p.rec_kind[r]), int(p.rec_flags[r])
        c0, c1 = int(p.rec_cell_base[r]), int(p.rec_cell_base[r + 1])
        key_image = f & RF_OLD_KEY and not f & RF_OLD_FULL
        if k == ord("I"):
            emit(r, [(c + 1, c, cell(c0 + c)) for c in range(nc)], "UPSERT", 0)
            continue
        if k not in (ord("U"), ord("D")):
            continue
        if (k == ord("U") and f & RF_NEW_PARTIAL) or (k == ord("D") and not f & (RF_OLD_FULL | RF_OLD_KEY)) or \
                (key_image and not identity_is_pk):
            invalid = min(invalid, r)
            continue
        old = None
        if f & RF_OLD_FULL:
            old = [(c, cell(c0 + c)) for c in pk_idx]
        elif f & RF_OLD_KEY:
            old = [(c, cell(c0 + q)) for q, c in enumerate(pk_idx)]
        if k == ord("D"):
            emit(r, [(c + 1, c, v) for c, v in old], "DELETE", 0)
            continue
        new = [cell(c1 - nc + c) for c in range(nc)]
        changed = old is not None and any(not cells_equal(v, new[c]) for c, v in old)
        if changed:
            emit(r, [(c + 1, c, v) for c, v in old], "DELETE", 0)
        emit(r, [(c + 1, c, new[c]) for c in range(nc)], "UPSERT", 1 if changed else 0)
    return dict(records=records, rows=rows, value=issues.get("value"), invalid=invalid)


def expected_copy_bigquery(rows_cells):
    """COPY rows given as [(tag, value)] per row (the oracle's per-row parse): UPSERT, no sequence field"""
    issues = {}
    rows = []
    for i, cells in enumerate(rows_cells):
        nc = len(cells)
        tagged = [(c + 1, c, v) for c, v in enumerate(cells)] + [(nc + 1, None, (2, "UPSERT"))]
        rows.append(row_bytes(tagged, issues, i))
    return dict(records=list(range(len(rows))), rows=rows, value=issues.get("value"), invalid=NONE64)
