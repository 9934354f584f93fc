"""Python restatement of the ClickHouse destination's RowBinary encoding (crates/etl-destinations/src/clickhouse):
write_events_inner / write_table_rows_inner (core.rs:489-521, :694-802) choosing the rows, expand_key_row / default_cell
(core.rs:920-997) widening key-only deletes, cell_to_clickhouse_value (encoding.rs:50-78) and rb_encode_nullable /
rb_encode_value / encode_to_row_binary (encoding.rs:176-273) writing the bytes, with the CDC columns cdc_operation /
cdc_lsn (core.rs:71-73, :505-509, :842-845).

Applied to a decoded batch's planes (canon.decode_cell values), `expected_rowbinary` gives what etl_dec_rowbinary_emit
must produce: rows, their bytes and the three issue reports.  The reference stops at an issue; the emitter carries on,
so a row with an issue follows the emitter's convention here (a NULL under a cleared flag writes nothing, an out-of-range
Date writes its day count), which keeps every later row's offsets comparable.
"""
from __future__ import annotations

import struct

from arrow_ref import json_display, numeric_display
from canon import CELL_ARRAY, CELL_NULL, RF_EVENT, RF_NEW_PARTIAL, RF_OLD_FULL, RF_OLD_KEY, decode_cell

NONE64, NONE32 = 2**64 - 1, 2**32 - 1
DATE32_MIN, DATE32_MAX = -25567, 120529        # 1900-01-01 ..= 2299-12-31 (encoding.rs:150-160)
CDC_OP = {ord("I"): b"INSERT", ord("U"): b"UPDATE", ord("D"): b"DELETE"}
# default_cell's wire width per decode class (ETL_K_*); String-like classes and arrays: one varint byte
DEFAULT_WIDTH = {1: 1, 3: 2, 4: 4, 5: 4, 7: 4, 10: 4, 6: 8, 8: 8, 12: 8, 13: 8, 14: 16}


# ------------------------------------------------------------------------------------------------ formatters
def varint(n: int) -> bytes:
    """rb_varint (encoding.rs:176-187): LEB128"""
    out = bytearray()
    while True:
        b = n & 0x7F
        n >>= 7
        if n == 0:
            out.append(b)
            return bytes(out)
        out.append(b | 0x80)


def hex_text(b: bytes) -> bytes:
    """bytes_to_hex (encoding.rs:162-172)"""
    return b.hex().encode()


def time_text(secs: int, nanos: int) -> bytes:
    """chrono NaiveTime's Display; nanos >= 10^9 is the leap second (:60)"""
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


def date32_ok(days: int) -> bool:
    return DATE32_MIN <= days <= DATE32_MAX


def uuid_wire(be: bytes) -> bytes:
    """u128::from_be_bytes, then the high u64 LE and the low u64 LE (encoding.rs:230-237)"""
    n = int.from_bytes(be, "big")
    return struct.pack("<QQ", n >> 64, n & NONE64)


def rb_string(b: bytes) -> bytes:
    return varint(len(b)) + b


# ------------------------------------------------------------------------------------------------ values
def value_bytes(tag: int, v, date_bad: list) -> bytes:
    """rb_encode_value of cell_to_clickhouse_value(cell) for a non-NULL cell of variant `tag` (ETL_CELL_*; the element
    kind for array elements, the numbering is the same).  A Date out of range appends its element index (None for a
    scalar) to date_bad and is written as its day count."""
    if tag == 1:
        return bytes([int(v)])
    if tag == 3:
        return struct.pack("<h", v)
    if tag == 4:
        return struct.pack("<i", v)
    if tag == 6:
        return struct.pack("<q", v)
    if tag == 5:
        return struct.pack("<I", v[1])
    if tag == "u64":                            # cdc_lsn (cdc_lsn_to_clickhouse_value, core.rs:71-73)
        return struct.pack("<Q", v)
    if tag == 7:
        return struct.pack("<I", v[1])
    if tag == 8:
        return struct.pack("<Q", v[1])
    if tag == 2:
        return rb_string(v.encode("utf-8"))
    if tag == 9:
        return rb_string(numeric_display(v).encode())
    if tag == 10:
        if not date32_ok(v[1]):
            date_bad.append(None)
        return struct.pack("<I", v[1] & NONE32)
    if tag == 11:
        return rb_string(time_text(v[1], v[2]))
    if tag in (12, 13):
        return struct.pack("<Q", (v[1] * 10**6 + v[2] // 1000) & NONE64)
    if tag == 14:
        return uuid_wire(bytes.fromhex(v[1]))
    if tag == 15:
        return rb_string(json_display(v[1]))
    if tag == 16:
        return rb_string(hex_text(v[1]))
    if tag == CELL_ARRAY:
        _, ek, elems = v
        out = [varint(len(elems))]
        for k, e in enumerate(elems):
            if e is None:
                out.append(b"\x01")
                continue
            bad = []
            out.append(b"\x00" + value_bytes(ek, e, bad))
            if bad:
                date_bad.append(k)
        return b"".join(out)
    raise ValueError(f"cell tag {tag} has no ClickHouse value")


def row_bytes(cells, flags, issues: dict, row: int) -> bytes:
    """encode_to_row_binary of one row: cells = [(tag, value) | ("default", kind)], flags = Nullable per column.
    Records the row's first Date32 / NULL issue in `issues` when none was recorded before."""
    out = []
    for c, (cell, nullable) in enumerate(zip(cells, flags)):
        m = b"\x00" if nullable else b""
        if cell[0] == "default":
            out.append(m + b"\x00" * DEFAULT_WIDTH.get(cell[1], 1))
            continue
        tag, v = cell
        if tag == CELL_NULL:
            if nullable:
                out.append(b"\x01")
            elif issues.get("null") is None:
                issues["null"] = (row, c, NONE32)
            continue
        bad = []
        out.append(m + value_bytes(tag, v, bad))
        if bad and issues.get("date") is None:
            issues["date"] = (row, c, NONE32 if bad[0] is None else bad[0])
    return b"".join(out)


# ------------------------------------------------------------------------------------------------ rows of a batch
def expand_key_row(key_cells, kinds, col_flags, pk):
    """expand_key_row (core.rs:944-962): primary-key columns take the key cells in order (NULL once they run out), other
    source-nullable non-array columns NULL, the rest default_cell"""
    it = iter(key_cells)
    out = []
    for c, kind in enumerate(kinds):
        if pk[c]:
            out.append(next(it, (CELL_NULL, None)))
        elif col_flags[c] & 1 and not kind & 0x20:
            out.append((CELL_NULL, None))
        else:
            out.append(("default", kind))
    return out


def pk_columns(schema, table_cols):
    """per replicated column: the stored TableSchema column (col_index) has a primary_key_ordinal_position"""
    return [table_cols[int(i)].get("pk") is not None for i in schema.col_index]


def expected_rowbinary(p, stream: bytes, schema_index: int, flags, table_cols):
    """etl_dec_rowbinary_emit of a streaming batch's schema version: dict(records, rows (bytes per row), date, null,
    partial).  table_cols = the stored TableSchema's columns (dicts with "pk") of the version's table."""
    sc = p.schemas[schema_index]
    heap = p.heap.tobytes()
    kinds = [int(k) for k in sc.col_kind]
    col_flags = [int(f) for f in sc.col_flags]
    pk = pk_columns(sc, table_cols)
    n = p.n_records if p.first_error[0] is None else p.first_error[0]
    nc = sc.n_cols

    def cell(i):
        tag = int(p.cell_tag[i])
        return tag, decode_cell(tag, int(p.cell_val[i]), int(p.cell_aux[i]), stream, heap)

    records, rows, issues, partial = [], [], {}, NONE64
    for r in range(n):
        if int(p.rec_schema[r]) != schema_index or not int(p.rec_flags[r]) & RF_EVENT:
            continue
        k, f = int(p.rec_kind[r]), int(p.rec_flags[r])
        c0, c1 = int(p.rec_cell_base[r]), int(p.rec_cell_base[r + 1])
        if k == ord("I"):
            cells = [cell(c0 + c) for c in range(nc)]
        elif k == ord("U"):
            if f & RF_NEW_PARTIAL:
                partial = min(partial, r)
                continue
            cells = [cell(c1 - nc + c) for c in range(nc)]
        elif k == ord("D") and f & RF_OLD_FULL:
            cells = [cell(c0 + c) for c in range(nc)]
        elif k == ord("D") and f & RF_OLD_KEY:
            cells = expand_key_row([cell(c0 + c) for c in range(sc.n_identity)], kinds, col_flags, pk)
        else:
            continue
        cells += [(2, CDC_OP[k].decode()), ("u64", int(p.rec_commit_lsn[r]))]
        rows.append(row_bytes(cells, flags, issues, len(rows)))
        records.append(r)
    return dict(records=records, rows=rows, date=issues.get("date"), null=issues.get("null"), partial=partial)


def expected_copy_rowbinary(rows_cells, flags):
    """COPY rows given as [(tag, value)] per row (the oracle's per-row parse): INSERT, LSN 0"""
    issues = {}
    rows = [row_bytes(list(cells) + [(2, "INSERT"), ("u64", 0)], flags, issues, i) for i, cells in enumerate(rows_cells)]
    return dict(records=list(range(len(rows))), rows=rows, date=issues.get("date"), null=issues.get("null"), partial=NONE64)


def create_table_flags(kinds, col_flags):
    """the Nullable wrappers build_create_table_sql gives a table: source-nullable non-array columns; the CDC columns
    are not nullable"""
    return [bool(f & 1) and not k & 0x20 for k, f in zip(kinds, col_flags)] + [False, False]
