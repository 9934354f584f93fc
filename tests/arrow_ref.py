"""Python restatements of the text the reference's Arrow encoders produce for Numeric, Json and array columns
(crates/etl-destinations/src/iceberg/encoding.rs: cell_to_string, build_list_array and its builders), and the expected
columns of etl_dec_arrow_emit with ETL_ARROW_ALL_COLUMNS built from a decoded batch's planes.

* numeric_display: PgNumeric's Display (crates/etl/src/conversions/numeric.rs:503-590).
* json_display: serde_json::Value's Display as the etl crate builds serde_json (arbitrary_precision, no
  preserve_order): compact, keys sorted by their UTF-8 bytes, the last of duplicate keys wins, numbers verbatim,
  strings escaped the serde_json way.  Third-party behaviour: parity unpinned (DESIGN §5).
"""
from __future__ import annotations

import json
import struct

import numpy as np

from canon import decode_cell

(A_UNSUP, A_BOOL, A_I32, A_I64, A_F32, A_F64, A_UTF8, A_LBIN, A_DATE32, A_TIME64, A_TS, A_TSTZ, A_UUID, A_LIST) = range(14)
ALL_COLUMNS = 0x100
KIND2ARROW = {1: A_BOOL, 2: A_UTF8, 3: A_I32, 4: A_I32, 5: A_I64, 6: A_I64, 7: A_F32, 8: A_F64, 9: A_UTF8, 10: A_DATE32, 11: A_TIME64,
              12: A_TS, 13: A_TSTZ, 14: A_UUID, 15: A_UTF8, 16: A_LBIN}


# ------------------------------------------------------------------------------------------------ Numeric
def numeric_display(num) -> str:
    """num = canon.numeric_from_heap's tuple: ("numeric", "NaN" | "Infinity" | "-Infinity") or
    ("numeric", sign, weight, scale, digits)"""
    if len(num) == 2:
        return num[1]
    _, sign, weight, scale, digits = num[:5]
    if not digits:
        return "0"

    def group(d):
        return digits[d] if 0 <= d < len(digits) else 0
    out = "-" if sign == "-" else ""
    if weight < 0:
        out += "0"
    else:
        for d in range(weight + 1):
            g = "%04d" % group(d)
            out += (g.lstrip("0") or "0") if d == 0 else g
    if scale > 0:
        out += "."
        rem, d = scale, weight + 1
        while rem > 0:
            take = min(4, rem)
            out += ("%04d" % group(d))[:take]
            rem -= take
            d += 1
    return out


def numeric_bytes(kind: int, sign: int, weight: int, scale: int, digits) -> bytes:
    """the heap entry of a numeric (etl_numeric_hdr + little-endian int16 digits)"""
    return struct.pack("<BBhHH", kind, sign, weight, scale, len(digits)) + struct.pack("<%dh" % len(digits), *digits)


# ------------------------------------------------------------------------------------------------ Json
class _Num(str):
    """a JSON number kept as its text (arbitrary_precision)"""


def _last_wins(pairs):
    d = {}
    for k, v in pairs:
        d[k] = v            # a repeated key keeps its first place in a dict, but order is re-derived when dumping
    return d


def _esc(s: str) -> str:
    out = ['"']
    for ch in s:
        c = ord(ch)
        if ch == '"':
            out.append('\\"')
        elif ch == "\\":
            out.append("\\\\")
        elif ch in "\b\f\n\r\t":
            out.append({"\b": "\\b", "\f": "\\f", "\n": "\\n", "\r": "\\r", "\t": "\\t"}[ch])
        elif c < 0x20:
            out.append("\\u%04x" % c)
        else:
            out.append(ch)
    out.append('"')
    return "".join(out)


def _dump(v, out):
    if v is None:
        out.append("null")
    elif v is True:
        out.append("true")
    elif v is False:
        out.append("false")
    elif isinstance(v, _Num):
        out.append(str(v))
    elif isinstance(v, str):
        out.append(_esc(v))
    elif isinstance(v, list):
        out.append("[")
        for i, x in enumerate(v):
            if i:
                out.append(",")
            _dump(x, out)
        out.append("]")
    else:
        out.append("{")
        for i, k in enumerate(sorted(v, key=lambda k: k.encode("utf-8"))):
            if i:
                out.append(",")
            out.append(_esc(k))
            out.append(":")
            _dump(v[k], out)
        out.append("}")


def json_display(text: bytes) -> bytes:
    v = json.loads(text.decode("utf-8"), parse_int=_Num, parse_float=_Num, object_pairs_hook=_last_wins)
    out = []
    _dump(v, out)
    return "".join(out).encode("utf-8")


# ------------------------------------------------------------------------------------------------ columns
def cell_text(value):
    """cell_to_string on a decoded cell (canon.decode_cell's form); None = null entry"""
    if isinstance(value, str):
        return value.encode("utf-8")
    if isinstance(value, tuple) and value[0] == "numeric":
        return numeric_display(value).encode()
    if isinstance(value, tuple) and value[0] == "json":
        return json_display(value[1])
    return None


def _time_us(value):
    return value[1] * 1000000 + value[2] // 1000


def element_value(child_type: int, value):
    """one list element: (valid, fixed value | bytes)"""
    if value is None:
        return False, None
    if child_type == A_BOOL:
        return True, bool(value)
    if child_type in (A_I32,):
        return True, int(value)
    if child_type == A_I64:
        return True, value[1] if isinstance(value, tuple) else int(value)
    if child_type in (A_F32, A_F64):
        return True, value[1]
    if child_type == A_DATE32:
        return True, value[1]
    if child_type in (A_TIME64, A_TS, A_TSTZ):
        return True, _time_us(value)
    if child_type == A_UUID:
        return True, bytes.fromhex(value[1])
    if child_type == A_LBIN:
        return True, value[1]
    return True, cell_text(value)


def selected_rows(p, schema_index: int, row_kinds: int):
    """(record index, first cell of the image) of every row the emitter selects, in stream order"""
    sc = p.schemas[schema_index]
    n = p.n_records if p.first_error[0] is None else p.first_error[0]
    rows = []
    for r in range(n):
        if int(p.rec_schema[r]) != schema_index or not int(p.rec_flags[r]) & 0x80:
            continue
        k, f = chr(int(p.rec_kind[r])), int(p.rec_flags[r])
        c0, c1 = int(p.rec_cell_base[r]), int(p.rec_cell_base[r + 1])
        if k == "I" and row_kinds & 1:
            rows.append((r, c0))
        elif k == "U" and row_kinds & 2 and not f & 4:
            rows.append((r, c1 - sc.n_cols))
        elif k == "D" and row_kinds & 4 and f & 1:
            rows.append((r, c0))
    return rows


def expected_formatted_columns(p, stream: bytes, schema_index: int, row_kinds: int):
    """expected Numeric / Json (Utf8) and array (List) columns of a schema version, from a decoded batch's planes:
    {column: ("utf8", valid[], offsets[], data) | ("list", valid[], list_offsets[], child_type, child_valid[], child)}
    where child is a list of element values (None for nulls) for fixed-width children and (offsets, data) for var-width"""
    sc = p.schemas[schema_index]
    heap = p.heap.tobytes()
    rows = selected_rows(p, schema_index, row_kinds)
    out = {}
    for c in range(sc.n_cols):
        kind = int(sc.col_kind[c])
        if kind not in (9, 15) and not kind & 0x20:
            continue
        cells = [decode_cell(int(p.cell_tag[c0 + c]), int(p.cell_val[c0 + c]), int(p.cell_aux[c0 + c]), stream, heap) for _, c0 in rows]
        if kind in (9, 15):
            texts = [cell_text(v) for v in cells]
            valid = np.array([t is not None for t in texts], dtype=bool)
            offs = np.zeros(len(texts) + 1, dtype=np.int64)
            offs[1:] = np.cumsum([len(t or b"") for t in texts])
            out[c] = ("utf8", valid, offs, b"".join(t or b"" for t in texts))
            continue
        ct = KIND2ARROW.get(kind & 0x1F, A_UNSUP)
        valid = np.array([isinstance(v, tuple) and v[0] == "array" for v in cells], dtype=bool)
        elems = [e for v in cells if isinstance(v, tuple) and v[0] == "array" for e in v[2]]
        loffs = np.zeros(len(cells) + 1, dtype=np.int64)
        loffs[1:] = np.cumsum([len(v[2]) if isinstance(v, tuple) and v[0] == "array" else 0 for v in cells])
        ev = [element_value(ct, e) for e in elems]
        cvalid = np.array([ok for ok, _ in ev], dtype=bool)
        if ct in (A_UTF8, A_LBIN):
            chunks = [x if ok else b"" for ok, x in ev]
            coffs = np.zeros(len(chunks) + 1, dtype=np.int64)
            coffs[1:] = np.cumsum([len(x) for x in chunks])
            child = (coffs, b"".join(chunks))
        else:
            child = [x if ok else None for ok, x in ev]
        out[c] = ("list", valid, loffs, ct, cvalid, child)
    return [r for r, _ in rows], out
