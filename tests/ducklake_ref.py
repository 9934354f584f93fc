"""Python restatement of the DuckLake destination's mutations, SQL-literal texts and batch identities
(crates/etl-destinations/src/ducklake):
* write_events_inner accumulating TableMutations (core.rs:715-836), validate_ducklake_replica_identity (:237-258) and
  key_row_from_updated_partial_row (:266-359);
* cell_to_sql_literal / array_cell_to_sql_literal / float_literal / encode_hex (encoding.rs:28-272) and
  table_row_to_sql_literal_ref, delete_predicate_from_row (batches.rs:1099-1186), update_assignments_from_partial_row
  (:1189-1269), delete_predicate_from_copy_row (:1338-1371);
* BatchIdHasher (FNV-1a 64, :196-224) fed the way Rust's Hash feeds it, build_mutation_batch_identity (:1272-1316),
  build_copy_batch_identity (:1319-1336), retain_mutations_after_sequence_key (:806-820) and the chunks of
  prepare_mutation_table_batches (:594-622).

Applied to a decoded batch's planes (canon.decode_cell values), `expected_ducklake` gives what etl_dec_ducklake_emit
must produce.  Rust's shortest float digits are taken to be Python's repr digits (no Rust toolchain checked that);
pg_escape's quote_literal is restated from PostgreSQL's rule (its source is not in the reference).
"""
from __future__ import annotations

import math
import struct
from decimal import Decimal

from arrow_ref import json_display, numeric_display
from bigquery_ref import date_text, uuid_text
from canon import CELL_ARRAY, CELL_MISSING, CELL_NULL, RF_EVENT, RF_NEW_PARTIAL, RF_OLD_FULL, RF_OLD_KEY, decode_cell

NONE64 = 2**64 - 1
INSERT, UPDATE, UPDATE_PARTIAL, REPLACE, DELETE, MF_ARRAY = 1, 2, 3, 4, 5, 0x80
REJ_UPDATE_NO_IDENTITY, REJ_DELETE_NO_IDENTITY, REJ_DELETE_NO_OLD_ROW, REJ_PARTIAL_KEY_MISSING = 1, 2, 3, 4
CHUNK = 16                                    # CDC_MUTATION_BATCH_SIZE
KIND_WORD = {INSERT: "insert", UPDATE: "update", UPDATE_PARTIAL: "update", REPLACE: "replace", DELETE: "delete"}


# ------------------------------------------------------------------------------------------------ FNV-1a 64 as Rust's Hash feeds it
class Hasher:
    def __init__(self):
        self.h = 0xCBF29CE484222325

    def write(self, b: bytes):
        h = self.h
        for x in b:
            h = ((h ^ x) * 0x100000001B3) & NONE64
        self.h = h

    def str(self, s):
        self.write(s.encode() if isinstance(s, str) else s)
        self.write(b"\xff")

    def u64(self, v: int):
        self.write(struct.pack("<Q", v))


def fnv1a64(b: bytes) -> int:
    h = Hasher()
    h.write(b)
    return h.h


# ------------------------------------------------------------------------------------------------ literals
def quote_literal(s: str) -> str:
    body = s.replace("'", "''").replace("\\", "\\\\")
    return ("E'" if "\\" in s else "'") + body + "'"


def f64_display(bits: int) -> str:
    """Rust's Display of a finite double: shortest round-trip digits laid out positionally"""
    x = struct.unpack("<d", struct.pack("<Q", bits))[0]
    if x == 0:
        return "-0" if bits >> 63 else "0"
    sign, digits, exp = Decimal(repr(x)).as_tuple()
    digits = list(digits)
    while digits[-1] == 0:
        digits.pop()
        exp += 1
    d = "".join(map(str, digits))
    n, p = len(d), len(d) + exp
    body = "0." + "0" * (-p) + d if p <= 0 else (d + "0" * (p - n) if p >= n else d[:p] + "." + d[p:])
    return ("-" if sign else "") + body


def f32_as_f64_bits(bits32: int) -> int:
    return struct.unpack("<Q", struct.pack("<d", struct.unpack("<f", struct.pack("<I", bits32))[0]))[0]


def float_literal(bits64: int, is_double: bool) -> str:
    x = struct.unpack("<d", struct.pack("<Q", bits64))[0]
    t = "DOUBLE" if is_double else "FLOAT"
    if math.isnan(x):
        return f"CAST('NaN' AS {t})"
    if math.isinf(x):
        return f"CAST('{'-' if x < 0 else ''}Infinity' AS {t})"
    return f64_display(bits64)


def time6(secs: int, nanos: int) -> str:
    """chrono's %H:%M:%S%.6f; nanos >= 10^9 is a leap second (:60)"""
    sec = secs % 60
    if nanos >= 10**9:
        sec += 1
        nanos -= 10**9
    return "%02d:%02d:%02d.%06d" % (secs // 3600, secs // 60 % 60, sec, nanos // 1000)


def timestamp6(secs: int, nanos: int) -> str:
    days, sod = divmod(secs, 86400)
    return date_text(days).decode() + " " + time6(sod, nanos)


def value_literal(tag: int, v) -> str:
    """cell_to_sql_literal of a decode_cell value"""
    if tag == CELL_NULL or v is None:
        return "NULL"
    if tag == 1:
        return "TRUE" if v else "FALSE"
    if tag in (3, 4, 6):
        return str(v)
    if tag == 5:
        return str(v[1])
    if tag == 7:
        return float_literal(f32_as_f64_bits(v[1]), False)
    if tag == 8:
        return float_literal(v[1], True)
    if tag == 2:
        return quote_literal(v)
    if tag == 9:
        return quote_literal(numeric_display(v))
    if tag == 10:
        return "DATE '%s'" % date_text(v[1]).decode()
    if tag == 11:
        return "TIME '%s'" % time6(v[1], v[2])
    if tag == 12:
        return "TIMESTAMP '%s'" % timestamp6(v[1], v[2])
    if tag == 13:
        return "TIMESTAMPTZ '%s+00:00'" % timestamp6(v[1], v[2])
    if tag == 14:
        return "CAST('%s' AS UUID)" % uuid_text(v[1]).decode()
    if tag == 15:
        return "CAST(%s AS JSON)" % quote_literal(json_display(v[1]).decode("utf-8"))
    if tag == 16:
        return "from_hex('%s')" % v[1].hex().upper()
    if tag == CELL_ARRAY:
        _, ek, elems = v
        return "[" + ", ".join("NULL" if e is None else value_literal(ek, e) for e in elems) + "]"
    raise ValueError(tag)


def row_text(cells) -> str:
    return "(" + ", ".join(value_literal(t, v) for t, v in cells) + ")"


def predicate_text(named_cells) -> str:
    """[(quoted name, (tag, value))] in schema order"""
    return " AND ".join(f"{n} IS NULL" if t == CELL_NULL else f"{n} = {value_literal(t, v)}" for n, (t, v) in named_cells)


def assignments(names, cells):
    """update_assignments_from_partial_row: [(index, literal)] of the present columns"""
    return [(c, value_literal(t, v)) for c, (t, v) in enumerate(cells) if t != CELL_MISSING]


def key_row_from_partial(cells, identity):
    """key_row_from_updated_partial_row: the identity cells of a partial row, None when one is missing"""
    out = []
    for c, (t, v) in enumerate(cells):
        if identity[c]:
            if t == CELL_MISSING:
                return None
            out.append((t, v))
    return out


# ------------------------------------------------------------------------------------------------ mutations of a batch
def expected_ducklake(p, stream: bytes, schema_index: int, names):
    """etl_dec_ducklake_emit of a streaming batch's schema version"""
    sc = p.schemas[schema_index]
    heap = p.heap.tobytes()
    nc = sc.n_cols
    identity = [bool(int(f) & 2) for f in sc.col_flags]
    id_cols = [c for c in range(nc) if identity[c]]
    n = p.n_records if p.first_error[0] is None else p.first_error[0]

    def cell(i):
        tag = int(p.cell_tag[i])
        return tag, decode_cell(tag, int(p.cell_val[i]), int(p.cell_aux[i]), stream, heap)

    out = dict(kinds=[], records=[], texts=([], [], []), seg=[], start=[], commit=[], tx=[], asg=[],
               rejected=NONE64, reason=0, empty=NONE64, mixed=0, n_cols=nc)
    seg, seg_flags = 0, {}

    def push(r, kind, row=None, pred=None, asg=None):
        arr = row is not None and any(t == CELL_ARRAY for t, _ in row)
        out["kinds"].append(kind | (MF_ARRAY if arr else 0))
        out["records"].append(r)
        out["texts"][0].append(row_text(row) if row is not None else "")
        out["texts"][1].append(pred if pred is not None else "")
        out["texts"][2].append(", ".join(f"{names[c]} = {a}" for c, a in asg) if asg is not None else "")
        out["asg"].append(asg)
        out["seg"].append(seg)
        out["start"].append(int(p.rec_start_lsn[r]))
        out["commit"].append(int(p.rec_commit_lsn[r]))
        out["tx"].append(int(p.rec_tx_ordinal[r]))

    def reject(r, why):
        if out["rejected"] == NONE64:
            out["rejected"], out["reason"] = r, why

    for r in range(n):
        k, f = int(p.rec_kind[r]), int(p.rec_flags[r])
        if not f & RF_EVENT:
            continue
        if k == ord("T"):
            seg += 1
            continue
        if k not in (ord("I"), ord("U"), ord("D")):
            continue
        if int(p.rec_schema[r]) != schema_index:
            if int(p.rec_rel[r]) == sc.table_id:
                seg_flags[seg] = seg_flags.get(seg, 0) | 2
            continue
        seg_flags[seg] = seg_flags.get(seg, 0) | 1
        c0, c1 = int(p.rec_cell_base[r]), int(p.rec_cell_base[r + 1])
        has_old = bool(f & (RF_OLD_FULL | RF_OLD_KEY))
        if f & RF_OLD_FULL:
            old = [(names[c], cell(c0 + c)) for c in id_cols]
        elif f & RF_OLD_KEY:
            old = [(names[c], cell(c0 + q)) for q, c in enumerate(id_cols)]
        else:
            old = None
        if k == ord("I"):
            push(r, INSERT, row=[cell(c0 + c) for c in range(nc)])
            continue
        if not id_cols:
            reject(r, REJ_UPDATE_NO_IDENTITY if k == ord("U") else REJ_DELETE_NO_IDENTITY)
            continue
        if k == ord("D"):
            if old is None:
                reject(r, REJ_DELETE_NO_OLD_ROW)
            else:
                push(r, DELETE, pred=predicate_text(old))
            continue
        new0 = c1 - nc if has_old else c0
        new = [cell(new0 + c) for c in range(nc)]
        if not f & RF_NEW_PARTIAL:
            if has_old:
                push(r, UPDATE, row=new, pred=predicate_text(old))
            else:
                push(r, REPLACE, row=new, pred=predicate_text([(names[c], new[c]) for c in id_cols]))
            continue
        if not has_old:
            key = key_row_from_partial(new, identity)
            if key is None:
                reject(r, REJ_PARTIAL_KEY_MISSING)
                continue
            old = [(names[c], kv) for c, kv in zip(id_cols, key)]
        asg = assignments(names, new)
        if not asg and out["empty"] == NONE64:
            out["empty"] = r
        push(r, UPDATE_PARTIAL, pred=predicate_text(old), asg=asg)
    out["mixed"] = int(any(v == 3 for v in seg_flags.values()))
    return out


def expected_copy_ducklake(rows_cells, names, pk):
    """COPY rows given as [(tag, value)] per row: INSERTs, predicate = delete_predicate_from_copy_row"""
    out = dict(kinds=[], records=[], texts=([], [], []), rejected=NONE64, reason=0, empty=NONE64, mixed=0)
    for i, cells in enumerate(rows_cells):
        out["kinds"].append(INSERT | (MF_ARRAY if any(t == CELL_ARRAY for t, _ in cells) else 0))
        out["records"].append(i)
        out["texts"][0].append(row_text(cells))
        out["texts"][1].append(predicate_text([(names[c], cv) for c, cv in enumerate(cells) if pk[c]]))
        out["texts"][2].append("")
    return out


# ------------------------------------------------------------------------------------------------ identities
def retained(want, last_key):
    """retain_mutations_after_sequence_key: indices of the mutations whose (commit_lsn, tx_ordinal) > last_key"""
    idx = range(len(want["records"]))
    if last_key is None:
        return list(idx)
    return [m for m in idx if (want["commit"][m], want["tx"][m]) > tuple(last_key)]


def mutation_fingerprint(want, table_name: bytes, ms) -> int:
    h = Hasher()
    h.str("mutation")
    h.str(table_name)
    for m in ms:
        h.u64(want["start"][m])
        h.u64(want["commit"][m])
        kind = want["kinds"][m] & 0x7F
        h.str(KIND_WORD[kind])
        if kind == INSERT:
            h.str(want["texts"][0][m])
        elif kind == DELETE:
            h.str(want["texts"][1][m])
        elif kind in (UPDATE, REPLACE):
            h.str(want["texts"][1][m])
            h.str(want["texts"][0][m])
        else:                                               # hash_partial_table_row_ref
            h.str(want["texts"][1][m])
            h.u64(want["n_cols"])
            for c, a in want["asg"][m]:
                h.u64(c)
                h.str(a)
    return h.h


def sub_batches(want, table_name: bytes, last_key=None):
    """[(first mutation, count, fingerprint)]: the kept mutations of each truncate-free run in chunks of 16"""
    kept = retained(want, last_key)
    out, cur, cur_seg = [], [], None
    for m in kept:
        if cur and (want["seg"][m] != cur_seg or len(cur) == CHUNK):
            out.append(cur)
            cur = []
        cur.append(m)
        cur_seg = want["seg"][m]
    if cur:
        out.append(cur)
    return [(ms[0], len(ms), mutation_fingerprint(want, table_name, ms)) for ms in out]


def batch_id(want, sub) -> str:
    first, n, fp = sub
    return "mutation:%016x:%016x:%016x" % (want["start"][first], want["commit"][first + n - 1], fp)


def copy_fingerprint(want, table_name: bytes) -> int:
    h = Hasher()
    h.str("copy")
    h.str(table_name)
    for pred, row in zip(want["texts"][1], want["texts"][0]):
        h.str(pred)
        h.str(row)
    return h.h
